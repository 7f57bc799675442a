"""Autoregressive text generation from a ``GPT2Engine``'s weights, on a KV cache.

``GPT2Generator`` decodes S sequences in lockstep from the engine's bf16 compute copy (``params.w16``), in place: no
copy of the weights, and none of the engine's activations, logits, gradients, optimizer state or inputs is touched --
the training step's CUDA graph owns those.  It keeps its own buffers for S rows and one KV cache per layer
(bf16 [S, max_len, 2, H, 64], ``n_layer * S * max_len * 2 * C`` elements in all), allocated on first use and kept.

One decode step is: ``embedding_decode`` -> per layer {LayerNorm, qkv GEMM, ``attention_decode`` (writes this position's
k / v into the cache), proj GEMM + residual, LayerNorm, fc GEMM + GELU, fc2 GEMM + residual} -> final LayerNorm -> logits
GEMM -> ``sample_tokens``, which also moves the shared position (a device int32) on.  No host argument changes from one
step to the next, so on CUDA the step is captured once per ``generate`` call as a CUDA graph and replayed for every
token; the prompt is fed through the same step (``sample_tokens`` forces the prompt's tokens), so a prefill needs no
second code path.  The GEMMs are the engine's (``TransformerEngine._linear``: wgmma, or cuBLAS with ``--gemm cublas``)
with a fixed tile width, so a sequence's logits do not depend on how many sequences are decoded with it.
"""
from __future__ import annotations

from typing import Callable, Optional

import torch

DECODE_BLOCK_N = 128      # tile width of every decode GEMM: fixed, so a row's result never depends on S


def generation_seed(seed: int, step: int) -> int:
    """The sampling seed of the generation a worker started with ``--seed seed`` runs at ``step``."""
    return (seed * 0x9E3779B97F4A7C15 + step * 0xBF58476D1CE4E5B9 + 1) % (1 << 63)


class GPT2Generator:
    def __init__(self, engine, count: int, max_len: int):
        cfg = engine.cfg
        if count < 1:
            raise ValueError(f"count must be >= 1, not {count}")
        if not 1 <= max_len <= cfg.block_size:
            raise ValueError(f"max_len {max_len} must be in [1, block_size={cfg.block_size}]")
        if cfg.n_embd != cfg.n_head * 64:
            raise ValueError(f"decoding needs a head dim of 64, not {cfg.n_embd // cfg.n_head}")
        self.engine, self.cfg = engine, cfg
        self.S, self.max_len = int(count), int(max_len)
        self.F = engine.F
        self._bufs = None
        self.caches = None

    # ------------------------------------------------------------------ buffers
    def _alloc(self) -> None:
        if self._bufs is not None:
            return
        cfg, S, dev = self.cfg, self.S, self.engine.dev
        C, H, L = cfg.n_embd, cfg.n_head, self.max_len
        bf = dict(device=dev, dtype=torch.bfloat16)
        f32 = dict(device=dev, dtype=torch.float32)
        i64 = dict(device=dev, dtype=torch.int64)
        b = dict(x=torch.empty(S, C, **bf), res1=torch.empty(S, C, **bf), ln=torch.empty(S, C, **bf),
                 mean=torch.empty(S, **f32), rstd=torch.empty(S, **f32), qkv=torch.empty(S, 3 * C, **bf),
                 att=torch.empty(S, C, **bf), fc_pre=torch.empty(S, 4 * C, **bf), fc_act=torch.empty(S, 4 * C, **bf),
                 logits=torch.empty(S, cfg.padded_vocab, **bf),
                 part=torch.empty(self.F.decode_partials(S, H, L), **f32),
                 pos=torch.zeros(2, device=dev, dtype=torch.int32), tok=torch.zeros(S, **i64),
                 out=torch.zeros(S, L, **i64), prompt=torch.zeros(S, L, **i64))
        self._bufs = b
        self.caches = [torch.zeros(S, L, 2, H, 64, **bf) for _ in range(cfg.n_layer)]

    @property
    def logits(self) -> torch.Tensor:
        """bf16 [S, padded vocab]: the logits of the last decode step."""
        self._alloc()
        return self._bufs["logits"]

    def cache_bytes(self) -> int:
        return self.cfg.n_layer * self.S * self.max_len * 2 * self.cfg.n_embd * 2

    # ------------------------------------------------------------------ one decode step
    @torch.no_grad()
    def _step(self, prompt_len: int, temperature: float, top_k: int, seed: int, first_seq: int) -> None:
        F, P, e, b = self.F, self.engine.params, self.engine, self._bufs
        bn = DECODE_BLOCK_N
        x, res1, ln = b["x"], b["res1"], b["ln"]
        F.embedding_decode(b["tok"], P.w16("wte"), P.w16("wpe"), b["pos"], x)
        for i, cache in enumerate(self.caches):
            p = f"h{i}."
            e.layernorm_fwd(x, P.w16(p + "ln1_w"), P.w16(p + "ln1_b"), ln, b["mean"], b["rstd"])
            e._linear(ln, P.w16(p + "qkv_w"), b["qkv"], bias=P.w16(p + "qkv_b"), block_n=bn)
            F.attention_decode(b["qkv"], cache, b["pos"], b["att"], b["part"], self.cfg.n_head)
            e._linear(b["att"], P.w16(p + "proj_w"), res1, bias=P.w16(p + "proj_b"), residual=x, block_n=bn)
            e.layernorm_fwd(res1, P.w16(p + "ln2_w"), P.w16(p + "ln2_b"), ln, b["mean"], b["rstd"])
            e._linear(ln, P.w16(p + "fc_w"), b["fc_act"], bias=P.w16(p + "fc_b"), gelu=True, aux=b["fc_pre"],
                      block_n=bn)
            e._linear(b["fc_act"], P.w16(p + "fc2_w"), x, bias=P.w16(p + "fc2_b"), residual=res1, block_n=bn)
        e.layernorm_fwd(x, P.w16("lnf_w"), P.w16("lnf_b"), ln, b["mean"], b["rstd"])
        e._linear(ln, P.w16("wte"), b["logits"], block_n=bn)
        F.sample_tokens(b["logits"], self.cfg.vocab_size, b["tok"], b["out"], b["prompt"], prompt_len, b["pos"],
                        temperature, top_k, seed, first_seq)

    # ------------------------------------------------------------------ generation
    def _prompt_rows(self, prompt_ids) -> torch.Tensor:
        p = torch.as_tensor(prompt_ids, dtype=torch.int64).cpu()
        if p.dim() == 1:
            p = p.unsqueeze(0).expand(self.S, -1)
        if p.dim() != 2 or p.shape[0] != self.S or p.shape[1] < 1:
            raise ValueError(f"the prompt must be a non-empty list of token ids, or one such row per sequence "
                             f"({self.S}), not shape {tuple(p.shape)}")
        bad = p[(p < 0) | (p >= self.cfg.vocab_size)]
        if bad.numel():
            raise ValueError(f"prompt token id {int(bad[0])} is outside the vocabulary [0, {self.cfg.vocab_size})")
        return p.contiguous()

    @torch.no_grad()
    def generate(self, prompt_ids, n_tokens: int, temperature: float = 1.0, top_k: int = 0, seed: int = 0,
                 first_seq: int = 0, use_graph: Optional[bool] = None, progress: Optional[Callable[[int], None]] = None,
                 logits_out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """int64 [S, len(prompt) + n_tokens] (CPU): the prompt followed by ``n_tokens`` generated tokens per sequence.

        ``prompt_ids``: one list of token ids for every sequence, or one row per sequence.  ``temperature`` 0 is greedy;
        ``top_k`` 0 samples from the whole vocabulary.  Sequence s draws with the Philox counter (seed, first_seq + s,
        position), so its tokens do not depend on S.  ``use_graph`` (default: on CUDA) replays one captured step per
        token after a first eager one.  ``progress(tokens done)`` is called every 16 steps.  ``logits_out`` (optional,
        [S, steps, vocab]) receives every step's logits, the step at position p predicting position p + 1."""
        cfg = self.cfg
        prompt = self._prompt_rows(prompt_ids)
        P = prompt.shape[1]
        if n_tokens < 0:
            raise ValueError(f"n_tokens must be >= 0, not {n_tokens}")
        if P + n_tokens > self.max_len:
            raise ValueError(f"prompt ({P}) plus tokens ({n_tokens}) exceed this generator's max_len {self.max_len} "
                             f"(block_size {cfg.block_size})")
        if not temperature >= 0:
            raise ValueError(f"temperature must be >= 0, not {temperature}")
        if not 0 <= top_k <= cfg.vocab_size:
            raise ValueError(f"top_k must be in [0, {cfg.vocab_size}], not {top_k}")
        self._alloc()
        b = self._bufs
        steps = P + n_tokens - 1
        b["prompt"].zero_()
        b["prompt"][:, :P].copy_(prompt)
        b["out"].zero_()
        b["out"][:, 0].copy_(prompt[:, 0])
        b["tok"].copy_(prompt[:, 0])
        b["pos"].zero_()
        args = (P, float(temperature), int(top_k), int(seed), int(first_seq))
        if use_graph is None:
            use_graph = self.engine.dev.type == "cuda"
        graph = None
        for i in range(steps):
            if graph is not None:
                graph.replay()
            else:
                self._step(*args)
                if use_graph and i + 1 < steps:
                    # the first step ran eagerly (module loading, kernel attributes); capture the next one once
                    graph = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(graph):
                        self._step(*args)
            if logits_out is not None:
                logits_out[:, i].copy_(b["logits"][:, :cfg.vocab_size])
            if progress is not None and (i + 1) % 16 == 0:
                progress(i + 1)
        return b["out"][:, :P + n_tokens].cpu()
