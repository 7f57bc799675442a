"""Training-step driver for the hand-written engines: pinned-host input feed, CUDA-graph replay,
bucketed gradient all-reduce overlapped with backward, fused optimizer sweep, loss read-back.

One ``step()`` is exactly what BASELINE.json's samples/sec counts and what ``bench.py`` times:
H2D copy of this step's tokens from pinned memory -> forward -> backward (+ all-reduce) ->
AdamW -> D2H of the loss.  The reference operator has no training loop (SURVEY.md §2.6); this is the
launched workers' loop.
"""
from __future__ import annotations

import math
import os
import time
from typing import List, Optional

import torch
import torch.distributed as dist

from ..parallel.ddp import BucketAllReducer


class SyntheticTokens:
    """Synthetic token stream of the named shape, staged in pinned host memory (no dataset access)."""

    def __init__(self, vocab: int, batch: int, seq: int, n_batches: int = 8, seed: int = 0, pin: bool = True):
        g = torch.Generator().manual_seed(seed)
        self.batches = []
        for _ in range(n_batches):
            tok = torch.randint(0, vocab, (batch * seq,), generator=g, dtype=torch.int64)
            tgt = torch.roll(tok, -1)
            if pin and torch.cuda.is_available():
                tok, tgt = tok.pin_memory(), tgt.pin_memory()
            self.batches.append((tok, tgt))
        self.i = 0
        self.bytes_per_step = 2 * batch * seq * 8

    def next(self):
        b = self.batches[self.i % len(self.batches)]
        self.i += 1
        return b


def cosine_lr(step: int, base_lr: float, warmup: int = 10, total: int = 10000, min_ratio: float = 0.1) -> float:
    if step < warmup:
        return base_lr * (step + 1) / warmup
    t = min(1.0, (step - warmup) / max(1, total - warmup))
    return base_lr * (min_ratio + (1 - min_ratio) * 0.5 * (1 + math.cos(math.pi * t)))


class EngineTrainer:
    def __init__(self, engine, lr: float = 3e-4, weight_decay: float = 0.1, max_norm: float = 1.0,
                 use_graph: bool = True, allreduce: Optional[str] = None, group=None):
        self.engine = engine
        self.lr = lr
        self.weight_decay = weight_decay
        self.max_norm = max_norm
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.group = group
        self.step_count = 0
        self.cuda = engine.dev.type == "cuda"
        # rs (default): gradients are reduce-scattered to their owner rank by the kernels that produce them, over NVLink
        # peer memory; sharded AdamW; bf16 parameters all-gathered by multicast stores (parallel/symm.ShardedGradState).
        # mc: every contribution multicast to all ranks (round-1 path).  nccl: bucketed library all-reduce.
        backend = allreduce or os.environ.get("AITJ_ALLREDUCE", "rs")
        self.allreduce_backend = backend if self.world > 1 else "none"
        self.symm = None
        self.shard = None
        self.reducer = None
        if getattr(engine.params, "shard", None) is not None:
            engine.params.detach_shard()      # re-bound after a re-rendezvous: the old group's symmetric buffers go
        if self.world > 1 and backend == "rs" and self.cuda:
            from ..parallel.symm import ShardedGradState

            sh = ShardedGradState(engine.params, engine.dev, group)
            if sh.available:
                engine.params.attach_shard(sh)
                self.shard = sh
                self.allreduce_backend = "rs (wgrad GEMM epilogue red.add to the owner over NVLink peer memory, sharded " \
                                         "AdamW, multicast all-gather of bf16 parameters)"
                sh.barrier()
            else:
                self.allreduce_backend = f"nccl (rs unavailable: {sh.reason})"
                backend = "nccl"
        if self.world > 1 and backend == "mc" and self.cuda:
            # fused GEMM -> all-reduce: gradients are reduced through the NVSwitch multicast alias by the kernels
            # that produce them (parallel/symm.py); no gradient collective is launched at all
            from ..parallel.symm import SymmetricGradBuffer

            self.symm = SymmetricGradBuffer(engine.params.total, engine.dev, group)
            if self.symm.available:
                engine.params.attach_grad_buffer(self.symm.tensor, self.symm.multicast_ptr)
            else:
                self.allreduce_backend = f"nccl (mc unavailable: {self.symm.reason})"
                self.symm = None
                backend = "nccl"
        if self.world > 1 and self.symm is None and self.shard is None:
            self.reducer = BucketAllReducer(engine.params.g32, engine.grad_buckets(), group, backend)
        engine.grad_hook = self.reducer.hook if self.reducer else None
        if self.reducer is not None:
            reserve = int(os.environ.get("AITJ_DDP_RESERVE_SMS", "0"))
            if reserve > 0:
                from ..ops import functional as F

                engine.bwd_max_ctas = max(2, (F.num_sms() - reserve) // 2 * 2)
                engine.split_k.clear()
        # Without library collectives (1 GPU, or the fused multicast path) the whole step is ONE CUDA graph.  With
        # the NCCL reducer the step is a chain of graphs split where a gradient bucket becomes final; the bucket's
        # all-reduce is launched between two replays on the side stream (capturing NCCL itself deadlocked on
        # the 2-GPU box), so collectives overlap the next segment's math and nothing else is launched eagerly.
        self.use_graph = use_graph and self.cuda
        self.segmented = self.reducer is not None
        # NCCL mode: a bucket's all-reduce starts when its segment's kernels are done, and segments are separate
        # graphs -- each one joins the weight-gradient side stream at its end
        engine.segment_join = self.segmented
        self.seg_graphs = None
        self.graph: Optional[torch.cuda.CUDAGraph] = None
        self.loss_host = torch.zeros(1, dtype=torch.float32)
        if self.cuda:
            self.loss_host = self.loss_host.pin_memory()
        self.graph_error: Optional[str] = None
        self.launches_per_step = 0

    # ------------------------------------------------------------------ one step of device work
    def _device_step(self) -> None:
        e = self.engine
        e.forward()
        if self.symm is not None:
            self.symm.barrier()   # every peer finished zeroing its gradients (previous optimizer sweep)
        e.backward()
        if self.symm is not None:
            self.symm.barrier()   # every peer's multimem reductions of this step have landed
        if self.shard is not None:
            self.shard.barrier()  # every contribution to this rank's shard has landed
        if self.reducer:
            self.reducer.wait()
        self._optimizer()
        if self.shard is not None:
            # every rank's bf16 parameters have arrived (next forward) and every shard is zeroed (next backward)
            self.shard.barrier()

    def _optimizer(self) -> None:
        self.engine.optimizer_step(lr=self.lr, step=max(1, self.step_count), weight_decay=self.weight_decay,
                                   max_norm=self.max_norm, grad_div=float(self.world), use_dyn=True)

    def _capture_segments(self) -> None:
        """NCCL mode: [forward] [bwd head] [layer L-1] ... [layer 0] [tail] [optimizer] as separate graphs."""
        from ..ops import lib

        e = self.engine
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(2):
                self._device_step()
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        saved_hook, e.grad_hook = e.grad_hook, None
        parts = [((), e.forward)] + list(e.backward_segments()) + [(None, self._optimizer)]
        graphs = []
        pool = None
        before = lib.LAUNCHES
        try:
            for buckets, fn in parts:
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g, pool=pool):
                    fn()
                if pool is None:
                    pool = g.pool()
                graphs.append((buckets, g))
            self.seg_graphs = graphs
            self.launches_per_step = lib.LAUNCHES - before
        except Exception as ex:  # noqa: BLE001
            self.seg_graphs = None
            self.use_graph = False
            self.graph_error = f"{type(ex).__name__}: {ex}"
            torch.cuda.synchronize()
        finally:
            e.grad_hook = saved_hook

    def _replay_segments(self) -> None:
        for buckets, g in self.seg_graphs:
            if buckets is None:            # optimizer: every bucket must have been reduced
                self.reducer.wait()
            g.replay()
            for b in buckets or ():
                self.reducer.hook(b)

    def _capture(self) -> None:
        from ..ops import lib

        # warm-up on a side stream (allocator, cuDNN plans, NCCL channels) before capture
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(2):
                self._device_step()
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        before = lib.LAUNCHES
        g = torch.cuda.CUDAGraph()
        try:
            with torch.cuda.graph(g):
                self._device_step()
            self.graph = g
            self.launches_per_step = lib.LAUNCHES - before
        except Exception as ex:  # noqa: BLE001 - fall back to eager replay
            self.graph = None
            self.use_graph = False
            self.graph_error = f"{type(ex).__name__}: {ex}"
            torch.cuda.synchronize()

    def count_launches_eager(self) -> int:
        from ..ops import lib

        before = lib.LAUNCHES
        self._device_step()
        return lib.LAUNCHES - before

    # ------------------------------------------------------------------ public step
    def step(self, *host_inputs: torch.Tensor, read_loss: bool = True) -> Optional[float]:
        """``host_inputs``: this step's inputs in pinned host memory, in the order of ``engine.input_tensors()``
        (GPT-2: tokens, targets; BERT: tokens, token types, MLM labels)."""
        e = self.engine
        self.step_count += 1
        for dst, src in zip(e.input_tensors(), host_inputs):
            dst.copy_(src, non_blocking=True)
        e.set_step_scalars(cosine_lr(self.step_count, self.lr), self.step_count)
        if self.use_graph and self.segmented:
            if self.seg_graphs is None:
                self._capture_segments()
            if self.seg_graphs is not None:
                self._replay_segments()
            else:
                self._device_step()
        elif self.use_graph:
            if self.graph is None:
                self._capture()
                # the two warm-up passes + capture consumed optimizer steps on real data; that is fine for
                # synthetic-data benchmarking and is excluded from timing by the caller's warm-up
            if self.graph is not None:
                self.graph.replay()
            else:
                self._device_step()
        else:
            self._device_step()
        if not read_loss:
            return None
        self.loss_host.copy_(e.loss, non_blocking=True)
        if self.cuda:
            torch.cuda.current_stream().synchronize()
        return float(self.loss_host[0])

    def state_tensors(self) -> List[torch.Tensor]:
        return self.engine.params.state_tensors()
