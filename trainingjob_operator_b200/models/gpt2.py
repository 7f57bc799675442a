"""GPT-2 training engine written for H100: explicit forward/backward over preallocated buffers.

This is one of the benchmark workloads BASELINE.json names ("GPT-2 small DDP"); the reference
operator itself contains no model code (SURVEY.md §2.6).  There is no autograd tape and no tracing
compiler on the hot path: every Linear is the hand-written wgmma/TMA GEMM
(``ops/csrc/gemm_wgmma.cu``) with its bias / GELU / dGELU / residual epilogue fused, weight gradients
are split-K GEMMs that ``red.add`` straight into the flat fp32 gradient buffer, LayerNorm, embedding,
softmax-cross-entropy and AdamW are single-sweep kernels (``ops/csrc/fused_ops.cu``), and the whole
step is captured in one CUDA graph.  Only scaled-dot-product attention calls a library kernel
(cuDNN / flash through ``torch``), as the task allows for plain library ops.

``GPT2Reference`` is the plain-PyTorch model sharing the same weights, used by the numerics tests.
"""
from __future__ import annotations

import dataclasses
import math
from dataclasses import dataclass
from typing import List, Tuple

import torch
import torch.nn.functional as TF

from .engine import TransformerEngine
from .flat_params import FlatParams, ParamSpec


@dataclass
class GPT2Config:
    vocab_size: int = 50257
    n_layer: int = 12
    n_head: int = 12
    n_embd: int = 768
    block_size: int = 1024
    name: str = "gpt2-small"

    @property
    def padded_vocab(self) -> int:
        return (self.vocab_size + 127) // 128 * 128

    @staticmethod
    def small() -> "GPT2Config":
        return GPT2Config()

    @staticmethod
    def tiny() -> "GPT2Config":
        return GPT2Config(vocab_size=1000, n_layer=2, n_head=4, n_embd=256, block_size=128, name="gpt2-tiny")


# The GPT-2 models by the name workers and ``cmd/generate`` take (``--model``).  Every size has head dim 64, vocabulary
# 50257 (50304 padded) and block size 1024; ``gpt2-tiny`` is for tests.
GPT2_MODELS = {
    "gpt2": GPT2Config.small(),
    "gpt2-medium": GPT2Config(n_layer=24, n_head=16, n_embd=1024, name="gpt2-medium"),
    "gpt2-large": GPT2Config(n_layer=36, n_head=20, n_embd=1280, name="gpt2-large"),
    "gpt2-xl": GPT2Config(n_layer=48, n_head=25, n_embd=1600, name="gpt2-xl"),
    "gpt2-tiny": GPT2Config.tiny(),
}


def gpt2_config(name: str) -> GPT2Config:
    """A copy of the ``GPT2_MODELS`` entry ``name``."""
    return dataclasses.replace(GPT2_MODELS[name])


def gpt2_param_specs(cfg: GPT2Config) -> List[ParamSpec]:
    """Flat layout: embeddings, then each layer's four weight matrices, then ALL 1-D parameters (biases, LayerNorm)
    in one tail region -- so a layer's matrices are one contiguous gradient bucket and the small parameters can be
    reduced with a single kernel in multicast mode."""
    C, L = cfg.n_embd, cfg.n_layer
    specs = [ParamSpec("wte", (cfg.padded_vocab, C), True), ParamSpec("wpe", (cfg.block_size, C), True, std=0.01)]
    pstd = 0.02 / math.sqrt(2 * L)
    for i in range(L):
        p = f"h{i}."
        specs += [ParamSpec(p + "qkv_w", (3 * C, C), True), ParamSpec(p + "proj_w", (C, C), True, std=pstd),
                  ParamSpec(p + "fc_w", (4 * C, C), True), ParamSpec(p + "fc2_w", (C, 4 * C), True, std=pstd)]
    for i in range(L):
        p = f"h{i}."
        specs += [ParamSpec(p + "ln1_w", (C,), False, "ones"), ParamSpec(p + "ln1_b", (C,), False, "zeros"),
                  ParamSpec(p + "qkv_b", (3 * C,), False, "zeros"), ParamSpec(p + "proj_b", (C,), False, "zeros"),
                  ParamSpec(p + "ln2_w", (C,), False, "ones"), ParamSpec(p + "ln2_b", (C,), False, "zeros"),
                  ParamSpec(p + "fc_b", (4 * C,), False, "zeros"), ParamSpec(p + "fc2_b", (C,), False, "zeros")]
    specs += [ParamSpec("lnf_w", (C,), False, "ones"), ParamSpec("lnf_b", (C,), False, "zeros")]
    return specs


def flops_per_token(cfg: GPT2Config, T: int) -> float:
    """fwd+bwd matmul FLOPs per token (6*N for the dense layers incl. tied lm_head + causal attention)."""
    C, L = cfg.n_embd, cfg.n_layer
    dense = L * (3 * C * C + C * C + 8 * C * C) + cfg.padded_vocab * C
    attn = L * 2 * T * C * 0.5  # QK^T and PV, causal half
    return 6.0 * dense + 6.0 * attn


class GPT2Engine(TransformerEngine):
    """GPT-2 (pre-LayerNorm decoder, tied lm_head) on ``TransformerEngine``; ``doc_mask`` as described there."""

    def __init__(self, cfg: GPT2Config, batch_size: int, seq_len: int, device="cuda", seed: int = 0,
                 gemm_backend: str = "wgmma", causal: bool = True, doc_mask: bool = False):
        super().__init__(cfg, gpt2_param_specs(cfg), batch_size, seq_len, device, seed, gemm_backend, causal, doc_mask)
        C, M = cfg.n_embd, self.M
        bf = dict(device=self.dev, dtype=torch.bfloat16)
        f32 = dict(device=self.dev, dtype=torch.float32)
        self.x0 = torch.empty(M, C, **bf)
        self.lnf = torch.empty(M, C, **bf)
        self.lnf_mean = torch.empty(M, **f32)
        self.lnf_rstd = torch.empty(M, **f32)
        self.d_res = [torch.empty(M, C, **bf) for _ in range(2)]
        self.d_ln = torch.empty(M, C, **bf)
        # evaluation (eval_forward): fp64 (sum of NLL, tokens); the cross-entropy partials are allocated on first use
        self.eval_acc = torch.zeros(2, device=self.dev, dtype=torch.float64)
        self._xent_part = self._xent_tgt = None
        # multiple-choice scoring (score_forward): fp64 (correct, examples); its other buffers are allocated on first use
        self.choice_acc = torch.zeros(2, device=self.dev, dtype=torch.float64)
        self._score_bufs = None

    def input_tensors(self) -> List[torch.Tensor]:
        """Device tensors a step reads its inputs from, in the order the data source yields them."""
        if self.doc_mask:
            return [self.tok, self.tgt, self.doc_start]
        return [self.tok, self.tgt]

    # ------------------------------------------------------------------ forward / backward segments
    @torch.no_grad()
    def forward(self) -> torch.Tensor:
        """Consumes self.tok / self.tgt; fills self.loss (mean NLL) and leaves dlogits in self.logits."""
        self._trunk()
        self._linear(self.lnf, self.params.w16("wte"), self.logits)
        return self._loss(self.M)

    @torch.no_grad()
    def eval_forward(self) -> torch.Tensor:
        """Evaluation forward on self.tok / self.tgt (target -1: a padding row): the layers of ``forward``, then the logits
        GEMM with the cross-entropy in its epilogue, so the logits never reach memory.  Fills self.losses with the
        per-token NLL (0 for padding) and adds (sum of the NLL, tokens with a target) to the fp64 ``self.eval_acc``, which
        the caller zeroes.  Leaves the logits, gradients and optimizer state as they are."""
        if self.backend != "wgmma":
            raise ValueError(f"evaluation needs the wgmma GEMM backend (its fused cross-entropy epilogue), not "
                             f"{self.backend!r}")
        self._nll_forward(self.eval_acc)
        return self.eval_acc

    def _nll_forward(self, acc: torch.Tensor, doc_start: torch.Tensor = None) -> None:
        """The evaluation forward of ``eval_forward`` and ``score_forward``: self.losses <- the per-token NLL of
        self.tgt, acc += (sum of the NLL, tokens with a target).  ``doc_start``: see ``_trunk``."""
        F, P, cfg = self.F, self.params, self.cfg
        if self._xent_part is None:
            self._xent_part = torch.empty(self.M, F.xent_blocks(cfg.padded_vocab), 2, device=self.dev,
                                          dtype=torch.float32)
            self._xent_tgt = torch.empty(self.M, device=self.dev, dtype=torch.float32)
        # a training step captured in a CUDA graph owns the tensors the attention forward leaves behind: keep them
        kept = [(lb.att_in, lb.sdpa_ctx) for lb in self.layers]
        self._trunk(doc_start)
        for lb, (att_in, ctx) in zip(self.layers, kept):
            lb.att_in, lb.sdpa_ctx = att_in, ctx
        wte = P.w16("wte")
        F.gemm_xent(self.lnf, wte, self.tgt, cfg.vocab_size, self._xent_part, self._xent_tgt,
                    block_n=self._bn(self.M, wte.shape[0], f"fwd:{wte.shape[0]}x{wte.shape[1]}"))
        F.xent_finish(self._xent_part, self._xent_tgt, self.tgt, self.losses, acc)

    @torch.no_grad()
    def score_forward(self, doc_start: torch.Tensor, spans: torch.Tensor, labels: torch.Tensor, E: int) -> torch.Tensor:
        """Multiple-choice scoring (HellaSwag) of E examples whose completions are packed as documents into the rows of
        self.tok / self.tgt (``runtime.hellaswag``): ``doc_start`` (int32 [B*T]) marks the documents, ``spans`` (int32
        [E, 4, 2], device) holds the (first row, rows) of each completion's targets and ``labels`` (int32 [E], device)
        the right ending.  The forward of ``eval_forward`` with positions counted from each document's start and the
        wgmma attention under the document mask -- whatever attention training runs -- then ``choice_score``:
        ``self.choice_acc`` (fp64 [2], zeroed by the caller) += (correct, examples).  Returns the per-completion mean NLL
        (fp32 [E, 4]).  Leaves the logits, gradients, optimizer state and ``eval_acc`` as they are."""
        H = self.cfg.n_head
        why = [w for bad, w in ((self.backend != "wgmma", f"gemm_backend is {self.backend!r}, not 'wgmma'"),
                                (not self.causal, "it needs causal attention"),
                                (self.T % 128, f"the sequence length {self.T} is not a multiple of 128"),
                                (self.cfg.n_embd // H != 64, f"the head dim {self.cfg.n_embd // H} is not 64")) if bad]
        if why:
            raise ValueError("scoring packed completions runs the wgmma GEMMs and document-masked attention, which cannot "
                             "serve this engine: " + "; ".join(why))
        if not 1 <= E <= self.M // self.F.CHOICES:
            raise ValueError(f"E = {E} examples: a micro-batch of {self.M} positions holds 1 to "
                             f"{self.M // self.F.CHOICES}")
        if self._score_bufs is None:
            ds = self.doc_start if self.doc_start is not None else \
                torch.zeros(self.M, dtype=torch.int32, device=self.dev)
            self._score_bufs = (ds, torch.zeros(2, dtype=torch.float64, device=self.dev),
                                torch.empty(self.M // self.F.CHOICES, self.F.CHOICES, dtype=torch.float32,
                                            device=self.dev))
        ds, nll_acc, mean = self._score_bufs
        if doc_start is not ds:
            ds.copy_(doc_start.reshape(-1), non_blocking=True)
        # nll_acc only receives xent_finish's (sum of NLL, tokens), which scoring does not use: it is never read or zeroed
        self._nll_forward(nll_acc, ds)
        self.F.choice_score(self.losses, spans, labels, mean[:E], self.choice_acc)
        return mean[:E]

    def _trunk(self, doc_start: torch.Tensor = None) -> None:
        """Embeddings, the layers and the final LayerNorm: self.lnf from self.tok.  ``doc_start`` (int32 [B*T]): packed
        documents, each embedded from position 0 and attended to under the document mask by the wgmma kernels."""
        F, P = self.F, self.params
        if doc_start is None:
            F.embedding_fwd(self.tok, P.w16("wte"), P.w16("wpe"), self.x0, self.T)
        else:
            F.embedding_doc_fwd(self.tok, P.w16("wte"), P.w16("wpe"), doc_start, self.x0, self.T)
        x = self.x0
        for i, lb in enumerate(self.layers):
            p = f"h{i}."
            self.layernorm_fwd(x, P.w16(p + "ln1_w"), P.w16(p + "ln1_b"), lb.ln1, lb.ln1_mean, lb.ln1_rstd)
            self._linear(lb.ln1, P.w16(p + "qkv_w"), lb.qkv, bias=P.w16(p + "qkv_b"))
            if doc_start is None:
                self._attention_fwd(lb)
            else:
                self._attention_doc_fwd(lb, doc_start)
            self._linear(lb.att_in, P.w16(p + "proj_w"), lb.res1, bias=P.w16(p + "proj_b"), residual=x)
            self.layernorm_fwd(lb.res1, P.w16(p + "ln2_w"), P.w16(p + "ln2_b"), lb.ln2, lb.ln2_mean, lb.ln2_rstd)
            self._linear(lb.ln2, P.w16(p + "fc_w"), lb.fc_act, bias=P.w16(p + "fc_b"), gelu=True, aux=lb.fc_pre)
            self._linear(lb.fc_act, P.w16(p + "fc2_w"), lb.res2, bias=P.w16(p + "fc2_b"), residual=lb.res1)
            x = lb.res2
        self.layernorm_fwd(x, P.w16("lnf_w"), P.w16("lnf_b"), self.lnf, self.lnf_mean, self.lnf_rstd)

    @torch.no_grad()
    def _bwd_head(self) -> None:
        F, P = self.F, self.params
        dlogits = self.logits
        self._dgrad(dlogits, P.w16("wte"), self.d_ln)
        self._wgrad(dlogits, self.lnf, P.grad("wte"))
        self._d_cur, self._d_spare = self.d_res
        x_last = self.layers[-1].res2 if self.layers else self.x0
        last = len(self.layers) - 1
        self.layernorm_bwd(self.d_ln, x_last, P.w16("lnf_w"), self.lnf_mean, self.lnf_rstd, self._d_cur,
                           P.grad("lnf_w"), P.grad("lnf_b"), dxsum=P.grad(f"h{last}.fc2_b") if last >= 0 else None)
        if self.segment_join:
            self._join_wgrads()

    @torch.no_grad()
    def _bwd_layer(self, i: int) -> None:
        F, P = self.F, self.params
        d_res, spare = self._d_cur, self._d_spare
        lb = self.layers[i]
        p = f"h{i}."
        x_in = self.layers[i - 1].res2 if i > 0 else self.x0
        # the previous segment's weight-gradient GEMMs still read d_fc / d_qkv / the residual-gradient buffers that this
        # layer is about to overwrite
        self._join_wgrads()
        # MLP (fc2_b's gradient = colsum(d_res) was already produced by the LayerNorm-backward that made d_res)
        e_fc2 = self._wgrad(d_res, lb.fc_act, P.grad(p + "fc2_w"))
        self._dgrad(d_res, P.w16(p + "fc2_w"), self.d_fc, dgelu_aux=lb.fc_pre, colsum=P.grad(p + "fc_b"))
        self._wgrad(self.d_fc, lb.ln2, P.grad(p + "fc_w"))
        self._dgrad(self.d_fc, P.w16(p + "fc_w"), self.d_ln)
        self.layernorm_bwd(self.d_ln, lb.res1, P.w16(p + "ln2_w"), lb.ln2_mean, lb.ln2_rstd, spare,
                           P.grad(p + "ln2_w"), P.grad(p + "ln2_b"), dres=d_res, dxsum=P.grad(p + "proj_b"))
        d_res, spare = spare, d_res
        # attention
        self._wgrad(d_res, lb.att_in, P.grad(p + "proj_w"))
        self._dgrad(d_res, P.w16(p + "proj_w"), self.d_att)
        self._attention_bwd(lb, self.d_att, self.d_qkv, P.grad(p + "qkv_b"))
        self._wgrad(self.d_qkv, lb.ln1, P.grad(p + "qkv_w"))
        self._dgrad(self.d_qkv, P.w16(p + "qkv_w"), self.d_ln)
        if e_fc2 is not None:
            torch.cuda.current_stream().wait_event(e_fc2)     # `spare` is the buffer the fc2 weight gradient read
        self.layernorm_bwd(self.d_ln, x_in, P.w16(p + "ln1_w"), lb.ln1_mean, lb.ln1_rstd, spare,
                           P.grad(p + "ln1_w"), P.grad(p + "ln1_b"), dres=d_res,
                           dxsum=P.grad(f"h{i - 1}.fc2_b") if i > 0 else None)
        self._d_cur, self._d_spare = spare, d_res
        if self.segment_join:
            self._join_wgrads()

    @torch.no_grad()
    def _bwd_tail(self) -> None:
        F, P = self.F, self.params
        F.embedding_bwd(self.tok, self._d_cur, P.grad("wte"), P.grad("wpe"), self.T)
        P.push_small_grads()
        self._join_wgrads()

    # ------------------------------------------------------------------ buckets (for DDP)
    def grad_buckets(self) -> List[Tuple[str, int, int]]:
        """(name, start, end) slices of the flat gradient buffer in the order backward completes them."""
        P = self.params
        out = []
        for i in range(self.cfg.n_layer - 1, -1, -1):
            out.append((f"h{i}",) + P.range_of(f"h{i}.qkv_w", f"h{i}.fc2_w"))
        out.append(("emb",) + P.range_of("wte", "wpe"))
        first_small = "h0.ln1_w" if self.cfg.n_layer > 0 else "lnf_w"
        out.append(("small",) + P.range_of(first_small, "lnf_b"))
        return out


# ------------------------------------------------------------------------------------ reference
class GPT2Reference(torch.nn.Module):
    """Plain PyTorch GPT-2 (fp32) reading the engine's master weights; used for numerics checks."""

    def __init__(self, cfg: GPT2Config, params: FlatParams, causal: bool = True):
        super().__init__()
        self.cfg = cfg
        self.causal = causal
        self.w = torch.nn.ParameterDict({s.name.replace(".", "_"): torch.nn.Parameter(params.w32(s.name).clone())
                                         for s in params.specs})

    def p(self, name: str) -> torch.Tensor:
        return self.w[name.replace(".", "_")]

    def forward(self, tok: torch.Tensor, tgt: torch.Tensor, doc_start: torch.Tensor = None) -> torch.Tensor:
        """``doc_start`` ([B, T] or [B*T], see ``GPT2Engine``): token q attends to key k iff doc_start[q] <= k <= q."""
        cfg = self.cfg
        B, T = tok.shape
        C, H = cfg.n_embd, cfg.n_head
        mask = None
        if doc_start is not None:
            assert self.causal
            ds = doc_start.reshape(B, 1, T, 1).long()
            k = torch.arange(T, device=tok.device).view(1, 1, 1, T)
            q = torch.arange(T, device=tok.device).view(1, 1, T, 1)
            mask = (k >= ds) & (k <= q)                        # [B, 1, T, T], True = attend
        x = self.p("wte")[tok] + self.p("wpe")[:T]
        for i in range(cfg.n_layer):
            q = f"h{i}."
            h = TF.layer_norm(x, (C,), self.p(q + "ln1_w"), self.p(q + "ln1_b"))
            qkv = h @ self.p(q + "qkv_w").t() + self.p(q + "qkv_b")
            qh, kh, vh = [t.view(B, T, H, C // H).transpose(1, 2) for t in qkv.split(C, dim=-1)]
            if mask is None:
                a = TF.scaled_dot_product_attention(qh, kh, vh, is_causal=self.causal)
            else:
                a = TF.scaled_dot_product_attention(qh, kh, vh, attn_mask=mask)
            a = a.transpose(1, 2).reshape(B, T, C)
            x = x + a @ self.p(q + "proj_w").t() + self.p(q + "proj_b")
            h = TF.layer_norm(x, (C,), self.p(q + "ln2_w"), self.p(q + "ln2_b"))
            h = TF.gelu(h @ self.p(q + "fc_w").t() + self.p(q + "fc_b"), approximate="tanh")
            x = x + h @ self.p(q + "fc2_w").t() + self.p(q + "fc2_b")
        x = TF.layer_norm(x, (C,), self.p("lnf_w"), self.p("lnf_b"))
        logits = x @ self.p("wte")[:cfg.vocab_size].t()
        return TF.cross_entropy(logits.view(B * T, -1), tgt.view(-1))
