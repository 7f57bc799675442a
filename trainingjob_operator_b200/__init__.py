"""aitj-b200: a single-box, H100-native elastic training-job controller with the capabilities of
``elasticdeeplearning/trainingjob-operator`` (AITrainingJob CRD surface, restart / completion / failure
policies, leader election, orphan GC) plus live elastic rescale, and the DDP workers it launches
(hand-written sm_90a kernels: wgmma/TMA GEMM, fused LayerNorm / cross-entropy / AdamW).  See DESIGN.md."""

__version__ = "0.1.0"
