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

import math
import os
from dataclasses import dataclass
from typing import Dict, List, Tuple

import torch
import torch.nn.functional as TF

from .flat_params import FlatParams, ParamSpec


# per-shape kernel choices (kind:NxK -> (block_n, split_k)) that override the default (the 2-CTA cluster wherever a
# 256x256 cluster tile fits); tools/gemm_cfg_sweep.py measures candidates in the captured step.  None is set by default.
_DEFAULT_GEMM_CFG: Dict[str, Tuple[int, int]] = {}

_QKV_GATHER = os.environ.get("AITJ_QKV_GATHER", "1") != "0"
_FUSE_COLSUM = os.environ.get("AITJ_FUSE_COLSUM", "1") != "0"


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


class _LayerBufs:
    def __init__(self, M: int, C: int, dev):
        bf = dict(device=dev, dtype=torch.bfloat16)
        f32 = dict(device=dev, dtype=torch.float32)
        self.ln1 = torch.empty(M, C, **bf)
        self.ln1_mean = torch.empty(M, **f32)
        self.ln1_rstd = torch.empty(M, **f32)
        self.qkv = torch.empty(M, 3 * C, **bf)
        self.att = torch.empty(M, C, **bf)
        self.res1 = torch.empty(M, C, **bf)
        self.ln2 = torch.empty(M, C, **bf)
        self.ln2_mean = torch.empty(M, **f32)
        self.ln2_rstd = torch.empty(M, **f32)
        self.fc_pre = torch.empty(M, 4 * C, **bf)
        self.fc_act = torch.empty(M, 4 * C, **bf)
        self.res2 = torch.empty(M, C, **bf)
        self.sdpa_ctx = None
        self.att_in = self.att
        self.lse = None              # [B, H, T] fp32, only with the wgmma attention forward


class GPT2Engine:
    """Explicit fwd/bwd/optimizer for a fixed (B, T) micro-batch on one GPU.

    ``doc_mask=True`` trains on packed documents: a step also reads ``doc_start`` (int32 [B*T], the sequence-local index of
    the first token of each token's document) and a token attends only to earlier tokens of its own document.  Only the
    wgmma attention kernels implement that mask, so they are used for the forward and the backward, and an engine they
    cannot serve is refused at construction."""

    doc_mask = False
    doc_start = None

    def __init__(self, cfg: GPT2Config, batch_size: int, seq_len: int, device="cuda", seed: int = 0,
                 gemm_backend: str = "wgmma", causal: bool = True, doc_mask: bool = False):
        from ..ops import functional as F

        assert seq_len <= cfg.block_size and cfg.n_embd % 256 == 0
        if doc_mask:
            why = [w for bad, w in ((not causal, "it needs causal attention"),
                                    (seq_len % 128, f"the sequence length {seq_len} is not a multiple of 128"),
                                    (cfg.n_embd // cfg.n_head != 64, f"the head dim {cfg.n_embd // cfg.n_head} is not 64"),
                                    (gemm_backend != "wgmma", f"gemm_backend is {gemm_backend!r}, not 'wgmma'")) if bad]
            if why:
                raise ValueError("document-masked attention runs on the wgmma attention kernels only, which cannot serve "
                                 "this engine: " + "; ".join(why))
        self.F = F
        self.cfg = cfg
        self.B, self.T = batch_size, seq_len
        self.M = batch_size * seq_len
        self.dev = torch.device(device)
        self.backend = gemm_backend
        # attention forward: "cudnn" (PyTorch SDPA -> cuDNN flash kernel) or "wgmma" (our kernel, AITJ_ATTN=wgmma).
        self.attn_impl = os.environ.get("AITJ_ATTN", "cudnn")
        if self.attn_impl == "wgmma" and (seq_len % 128 or cfg.n_embd // cfg.n_head != 64 or gemm_backend != "wgmma"):
            self.attn_impl = "cudnn"
        # attention backward: "wgmma" (ops/csrc/attention_bwd_wgmma.cu: dq/dk/dv written straight into the packed d_qkv)
        # needs our forward's log-sum-exp, so it implies the wgmma forward; "cudnn" = library kernel + gather
        self.attn_bwd_impl = os.environ.get("AITJ_ATTN_BWD", "cudnn")
        if self.attn_impl != "wgmma":
            self.attn_bwd_impl = "cudnn"
        self.doc_mask = bool(doc_mask)
        if self.doc_mask:
            self.attn_impl = self.attn_bwd_impl = "wgmma"
        self._attn_delta = None
        self._dq_acc = None
        self._philox = torch.zeros((), dtype=torch.int64, device=device)
        # backward GEMMs may leave a few SMs to the gradient all-reduce kernels that run next to them (DDP): a
        # persistent grid of exactly #SMs CTAs needs a second wave as soon as a collective holds some SMs
        self.bwd_max_ctas = 0
        self.causal = causal
        self.params = FlatParams(gpt2_param_specs(cfg), self.dev, seed=seed)
        C, M, Vp = cfg.n_embd, self.M, cfg.padded_vocab
        with torch.no_grad():
            self.params.w32("wte")[cfg.vocab_size:].zero_()
            self.params.refresh_compute_copy()
        bf = dict(device=self.dev, dtype=torch.bfloat16)
        f32 = dict(device=self.dev, dtype=torch.float32)
        self.tok = torch.zeros(M, dtype=torch.int64, device=self.dev)
        self.tgt = torch.zeros(M, dtype=torch.int64, device=self.dev)
        if self.doc_mask:
            self.doc_start = torch.zeros(M, dtype=torch.int32, device=self.dev)
        self.x0 = torch.empty(M, C, **bf)
        self.layers = [_LayerBufs(M, C, self.dev) for _ in range(cfg.n_layer)]
        self.lnf = torch.empty(M, C, **bf)
        self.lnf_mean = torch.empty(M, **f32)
        self.lnf_rstd = torch.empty(M, **f32)
        self.logits = torch.empty(M, Vp, **bf)
        self.losses = torch.empty(M, **f32)
        self.loss = torch.zeros(1, **f32)
        # backward scratch
        self.d_res = [torch.empty(M, C, **bf) for _ in range(2)]
        self.d_ln = torch.empty(M, C, **bf)
        self.d_fc = torch.empty(M, 4 * C, **bf)
        self.d_qkv = torch.empty(M, 3 * C, **bf)
        self.d_att = torch.empty(M, C, **bf)
        # optimizer scalars
        self.sumsq = torch.zeros(1, **f32)
        self.dyn = torch.zeros(4, **f32)
        self._dyn_host = torch.zeros(4, dtype=torch.float32).pin_memory() if self.dev.type == "cuda" else None
        import os as _os

        # 2-CTA cluster GEMM: two 128x256 tiles sharing the B tile by TMA multicast (AITJ_GEMM_PAIR=0: single CTAs)
        self.pair = _os.environ.get("AITJ_GEMM_PAIR", "1") != "0"
        # per-GEMM kernel choice measured in the step (tools/gemm_cfg_sweep.py): "kind:NxK=block_n[/split_k]" entries,
        # block_n 512 = 2-CTA cluster, 256 / 128 = 1-CTA tiles; AITJ_GEMM_CFG overrides / extends the table
        self.gemm_cfg: Dict[str, Tuple[int, int]] = dict(_DEFAULT_GEMM_CFG)
        for item in filter(None, _os.environ.get("AITJ_GEMM_CFG", "").split(",")):
            k, v = item.split("=")
            bn, _, sk = v.partition("/")
            self.gemm_cfg[k.strip()] = (int(bn), int(sk or 0))
        # weight-gradient GEMMs on a side stream (AITJ_WGRAD_STREAM=0: in line); see _wgrad
        self.wgrad_stream = torch.cuda.Stream() if (self.dev.type == "cuda" and gemm_backend == "wgmma" and
                                                    _os.environ.get("AITJ_WGRAD_STREAM", "0") != "0") else None
        self._wgrad_done = None
        self.segment_join = False     # True: every backward segment joins the side stream (segments are separate graphs)
        self.grad_hook = None  # called as hook(name_of_bucket) when a gradient bucket is complete
        self._graph = None
        self.split_k: Dict[Tuple[int, int], int] = {}

    def input_tensors(self) -> List[torch.Tensor]:
        """Device tensors a step reads its inputs from, in the order the data source yields them."""
        if self.doc_mask:
            return [self.tok, self.tgt, self.doc_start]
        return [self.tok, self.tgt]

    # ------------------------------------------------------------------ GEMM front-ends
    def _linear(self, x, w, out, bias=None, residual=None, gelu=False, aux=None):
        F = self.F
        if self.backend == "wgmma":
            F.gemm(x, w, out, bias=bias, residual=residual, gelu=gelu, save_pre=gelu, aux=aux,
                   block_n=self._bn(x.shape[0], w.shape[0], f"fwd:{w.shape[0]}x{w.shape[1]}"))
            return out
        # library path (cuBLAS) + standalone elementwise kernels; numerics cross-check / fallback bench arm
        y = torch.addmm(bias, x, w.t()) if bias is not None else x @ w.t()
        if gelu:
            aux.copy_(y)
            F.gelu_fwd(aux, out)
        elif residual is not None:
            torch.add(y, residual, out=out)
        else:
            out.copy_(y)
        return out

    def _bn(self, m: int, n: int, key: str = "") -> int:
        """512 = 2-CTA cluster kernel when the problem has at least one full 256x256 cluster tile, else auto 1-CTA; a measured
        per-shape choice in ``gemm_cfg`` wins."""
        if key in self.gemm_cfg:
            return self.gemm_cfg[key][0]
        return 512 if self.pair and m >= 256 and n >= 256 else 0

    def _dgrad(self, dy, w, out, dgelu_aux=None, colsum=None, residual=None):
        """out[M,K] = dy[M,N] @ w[N,K]  (* gelu'(aux)) (+ residual: the gradient arriving over a skip connection);
        colsum (fp32[K], optional) += column sums of out."""
        F = self.F
        if self.backend == "wgmma":
            bn = self._bn(dy.shape[0], w.shape[1], f"dgrad:{w.shape[1]}x{w.shape[0]}")
            fused = colsum is not None and bn == 512 and _FUSE_COLSUM
            F.gemm(dy, w, out, b_mn=True, dgelu=dgelu_aux is not None, aux=dgelu_aux, residual=residual,
                   block_n=bn, max_ctas=self.bwd_max_ctas, colsum=colsum if fused else None)
            if colsum is not None and not fused:
                F.colsum(out, colsum)
            return out
        y = dy @ w
        if dgelu_aux is not None:
            F.gelu_bwd(dgelu_aux, y, out)
        elif residual is not None:
            torch.add(y, residual, out=out)
        else:
            out.copy_(y)
        if colsum is not None:
            F.colsum(out, colsum)
        return out

    def _wgrad(self, dy, x, dw):
        """dw[N,K] (fp32) += dy[M,N]^T @ x[M,K].

        Weight gradients are leaves of the backward graph: nothing in the backward chain reads them.  With
        ``wgrad_stream`` they are launched on a side stream behind an event on the producer of ``dy``, so the tail of a
        weight-gradient GEMM -- and, in the owner-sharded mode, the time its finished blocks need to drain over NVLink --
        is filled by the input-gradient GEMMs / LayerNorm / attention kernels of the chain.  Returns the event that marks
        its completion (``None`` when launched in line); ``_join_wgrads`` / explicit waits order later writers of ``dy``."""
        side = self.wgrad_stream
        if side is None:
            self._wgrad_now(dy, x, dw)
            return None
        main = torch.cuda.current_stream()
        ready = torch.cuda.Event()
        ready.record(main)
        side.wait_event(ready)
        with torch.cuda.stream(side):
            self._wgrad_now(dy, x, dw)
            done = torch.cuda.Event()
            done.record(side)
        self._wgrad_done = done
        return done

    def _join_wgrads(self) -> None:
        """The current stream waits for every weight-gradient GEMM launched so far (the side stream is in order)."""
        if self._wgrad_done is not None:
            torch.cuda.current_stream().wait_event(self._wgrad_done)
            self._wgrad_done = None

    def _wgrad_now(self, dy, x, dw):
        F = self.F
        if self.backend == "wgmma":
            key = (dw.shape[0], dw.shape[1])
            if getattr(dw, "is_multicast", False):
                # fused wgrad -> all-reduce: partial sums would each cross the switch, so no split-K; narrower tiles
                # keep the SMs busy instead
                tiles256 = ((dw.shape[0] + 127) // 128) * ((dw.shape[1] + 255) // 256)
                F.gemm(dy, x, dw, a_mn=True, b_mn=True, accumulate=True, split_k=1,
                       block_n=256 if tiles256 >= F.num_sms() else 128)
                return
            ck = f"wgrad:{dw.shape[0]}x{dw.shape[1]}"
            bn = self._bn(dw.shape[0], dw.shape[1], ck)
            sk = self.split_k.get(key)
            if sk is None:
                sk = self.gemm_cfg.get(ck, (0, 0))[1] or \
                    F.auto_split_k(dw.shape[0], dw.shape[1], dy.shape[0], block_n=bn if bn != 512 else 0, pair=(bn == 512))
                self.split_k[key] = sk
            F.gemm(dy, x, dw, a_mn=True, b_mn=True, accumulate=True, split_k=sk, block_n=bn,
                   max_ctas=self.bwd_max_ctas)
        else:
            dw.add_((dy.t() @ x).float())

    # ------------------------------------------------------------------ attention (library op)
    def _attention_fwd(self, lb: _LayerBufs):
        B, T, H = self.B, self.T, self.cfg.n_head
        D = self.cfg.n_embd // H
        if self.attn_impl == "wgmma":
            # hand-written flash-attention forward (ops/csrc/attention_wgmma.cu): reads the packed qkv in place,
            # writes [B*T, H*D] and the log-sum-exp the backward needs
            if lb.lse is None:
                lb.lse = torch.empty(B, H, T, device=self.dev, dtype=torch.float32)
            if self.doc_mask:
                self.F.attention_fwd(lb.qkv, lb.att, lb.lse, B, T, H, causal=self.causal, doc_start=self.doc_start)
            else:
                self.F.attention_fwd(lb.qkv, lb.att, lb.lse, B, T, H, causal=self.causal)
            lb.att_in = lb.att
            return
        qkv = lb.qkv.view(B, T, 3, H, D)
        q = qkv[:, :, 0].transpose(1, 2).detach().requires_grad_(True)
        k = qkv[:, :, 1].transpose(1, 2).detach().requires_grad_(True)
        v = qkv[:, :, 2].transpose(1, 2).detach().requires_grad_(True)
        with torch.enable_grad():
            o = TF.scaled_dot_product_attention(q, k, v, is_causal=self.causal)
        lb.sdpa_ctx = (q, k, v, o)
        ot = o.detach().transpose(1, 2)
        if ot.is_contiguous():
            lb.att_in = ot.reshape(B * T, H * D)     # cuDNN wrote [B,T,H,D] already: feed the GEMM in place
        else:
            lb.att.view(B, T, H, D).copy_(ot)
            lb.att_in = lb.att

    def _attention_bwd(self, lb: _LayerBufs, d_att: torch.Tensor, d_qkv: torch.Tensor, d_bias: torch.Tensor):
        """d_qkv <- SDPA backward; d_bias (the qkv bias gradient) += colsum(d_qkv), fused into the gather."""
        B, T, H = self.B, self.T, self.cfg.n_head
        D = self.cfg.n_embd // H
        if self.attn_bwd_impl == "wgmma":
            if self._dq_acc is None:
                self._attn_delta = torch.empty(B, H, T, device=self.dev, dtype=torch.float32)
                self._dq_acc = torch.zeros(B * T, H * D, device=self.dev, dtype=torch.float32)
            if self.doc_mask:
                self.F.attention_bwd(lb.qkv, lb.att, d_att, lb.lse, self._attn_delta, self._dq_acc, d_qkv, B, T, H,
                                     causal=self.causal, doc_start=self.doc_start)
            else:
                self.F.attention_bwd(lb.qkv, lb.att, d_att, lb.lse, self._attn_delta, self._dq_acc, d_qkv, B, T, H,
                                     causal=self.causal)
            self.F.colsum(d_qkv, d_bias)
            return
        do = d_att.view(B, T, H, D).transpose(1, 2)
        if self.attn_impl == "wgmma":
            # cuDNN's SDPA backward accepts our forward's output and log-sum-exp ([B,H,T,1], natural log)
            qkv5 = lb.qkv.view(B, T, 3, H, D)
            q, k, v = (qkv5[:, :, i].transpose(1, 2) for i in range(3))
            o4 = lb.att.view(B, T, H, D).transpose(1, 2)
            dq, dk, dv = torch.ops.aten._scaled_dot_product_cudnn_attention_backward(
                do, q, k, v, o4, lb.lse.view(B, H, T, 1), self._philox, self._philox, None, None, None, T, T, 0.0,
                self.causal)
        else:
            q, k, v, o = lb.sdpa_ctx
            dq, dk, dv = torch.autograd.grad(o, (q, k, v), do)
        if _QKV_GATHER:
            self.F.qkv_gather_colsum(dq, dk, dv, d_qkv, d_bias)
        else:   # A/B arm: three strided copies + a separate column reduction
            dst = d_qkv.view(B, T, 3, H, D)
            dst[:, :, 0].copy_(dq.transpose(1, 2))
            dst[:, :, 1].copy_(dk.transpose(1, 2))
            dst[:, :, 2].copy_(dv.transpose(1, 2))
            self.F.colsum(d_qkv, d_bias)
        lb.sdpa_ctx = None

    # ------------------------------------------------------------------ forward / backward
    @torch.no_grad()
    def forward(self) -> torch.Tensor:
        """Consumes self.tok / self.tgt; fills self.loss (mean NLL) and leaves dlogits in self.logits."""
        F, P, cfg = self.F, self.params, self.cfg
        F.embedding_fwd(self.tok, P.w16("wte"), P.w16("wpe"), self.x0, self.T)
        x = self.x0
        for i, lb in enumerate(self.layers):
            p = f"h{i}."
            F.layernorm_fwd(x, P.w16(p + "ln1_w"), P.w16(p + "ln1_b"), lb.ln1, lb.ln1_mean, lb.ln1_rstd)
            self._linear(lb.ln1, P.w16(p + "qkv_w"), lb.qkv, bias=P.w16(p + "qkv_b"))
            self._attention_fwd(lb)
            self._linear(lb.att_in, P.w16(p + "proj_w"), lb.res1, bias=P.w16(p + "proj_b"), residual=x)
            F.layernorm_fwd(lb.res1, P.w16(p + "ln2_w"), P.w16(p + "ln2_b"), lb.ln2, lb.ln2_mean, lb.ln2_rstd)
            self._linear(lb.ln2, P.w16(p + "fc_w"), lb.fc_act, bias=P.w16(p + "fc_b"), gelu=True, aux=lb.fc_pre)
            self._linear(lb.fc_act, P.w16(p + "fc2_w"), lb.res2, bias=P.w16(p + "fc2_b"), residual=lb.res1)
            x = lb.res2
        F.layernorm_fwd(x, P.w16("lnf_w"), P.w16("lnf_b"), self.lnf, self.lnf_mean, self.lnf_rstd)
        self._linear(self.lnf, P.w16("wte"), self.logits)
        F.softmax_xent(self.logits, self.tgt, self.losses, cfg.vocab_size, 1.0 / self.M)
        torch.sum(self.losses, dim=0, keepdim=True, out=self.loss)
        self.loss.mul_(1.0 / self.M)
        return self.loss

    @torch.no_grad()
    def backward(self) -> None:
        """Accumulates into the flat fp32 gradient buffer (zeroed by the optimizer sweep)."""
        hook = self.grad_hook
        for buckets, fn in self.backward_segments():
            fn()
            if hook:
                for b in buckets:
                    hook(b)

    def backward_segments(self):
        """Backward split at the points where a gradient bucket becomes final: [(finished buckets, callable)].
        The trainer captures each callable as its own CUDA graph and launches the bucket's all-reduce between
        replays, so library collectives stay outside the graphs while everything else is replayed."""
        segs = [((), self._bwd_head)]
        for i in range(len(self.layers) - 1, -1, -1):
            segs.append(((f"h{i}",), (lambda i=i: self._bwd_layer(i))))
        segs.append((("emb", "small"), self._bwd_tail))
        return segs

    @torch.no_grad()
    def _bwd_head(self) -> None:
        F, P = self.F, self.params
        dlogits = self.logits
        self._dgrad(dlogits, P.w16("wte"), self.d_ln)
        self._wgrad(dlogits, self.lnf, P.grad("wte"))
        self._d_cur, self._d_spare = self.d_res
        x_last = self.layers[-1].res2 if self.layers else self.x0
        last = len(self.layers) - 1
        F.layernorm_bwd(self.d_ln, x_last, P.w16("lnf_w"), self.lnf_mean, self.lnf_rstd, self._d_cur, P.grad("lnf_w"),
                        P.grad("lnf_b"), dxsum=P.grad(f"h{last}.fc2_b") if last >= 0 else None)
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
        F.layernorm_bwd(self.d_ln, lb.res1, P.w16(p + "ln2_w"), lb.ln2_mean, lb.ln2_rstd, spare,
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
        F.layernorm_bwd(self.d_ln, x_in, P.w16(p + "ln1_w"), lb.ln1_mean, lb.ln1_rstd, spare,
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

    # ------------------------------------------------------------------ optimizer
    def set_step_scalars(self, lr: float, step: int, beta1: float = 0.9, beta2: float = 0.95) -> None:
        """Refresh {lr, 1-b1^t, 1-b2^t} on the device (outside the captured graph)."""
        vals = [lr, 1.0 - beta1 ** step, 1.0 - beta2 ** step, 0.0]
        if self._dyn_host is not None:
            for i, v in enumerate(vals):
                self._dyn_host[i] = v
            self.dyn.copy_(self._dyn_host, non_blocking=True)
        else:
            self.dyn.copy_(torch.tensor(vals))

    @torch.no_grad()
    def optimizer_step(self, lr: float = 3e-4, step: int = 1, weight_decay: float = 0.1, max_norm: float = 1.0,
                       grad_div: float = 1.0, beta1: float = 0.9, beta2: float = 0.95, use_dyn: bool = False) -> None:
        F, P = self.F, self.params
        sh = P.shard
        if sh is not None:
            # owner-sharded: this rank holds the summed gradient of [lo, hi) only.  Clip on the global norm (partial
            # square sums exchanged by multicast store), AdamW on the shard, bf16 parameters stored into every rank's copy.
            lo, hi = sh.lo, sh.hi
            self.sumsq.zero_()
            if max_norm > 0 and hi > lo:
                F.sumsq(P.g32[lo:hi], self.sumsq)
            F.norm_share(sh.parts_mc, self.sumsq, sh.rank)
            sh.barrier()
            if hi > lo:
                F.adamw(P.p32[lo:hi], P.g32[lo:hi], P.m[lo:hi], P.v[lo:hi], sh.w_mc + 2 * lo, P.wd_mask[lo // 256:],
                        lr=lr, beta1=beta1, beta2=beta2, eps=1e-8, weight_decay=weight_decay, step=step,
                        sumsq_buf=sh.parts if max_norm > 0 else None, max_norm=max_norm, grad_div=grad_div,
                        zero_grad=True, dyn=self.dyn if use_dyn else None, sumsq_n=sh.world, p16_multicast=True)
            return
        if max_norm > 0:
            self.sumsq.zero_()
            F.sumsq(P.g32, self.sumsq)
        F.adamw(P.p32, P.g32, P.m, P.v, P.p16, P.wd_mask, lr=lr, beta1=beta1, beta2=beta2, eps=1e-8,
                weight_decay=weight_decay, step=step, sumsq_buf=self.sumsq if max_norm > 0 else None,
                max_norm=max_norm, grad_div=grad_div, zero_grad=True, dyn=self.dyn if use_dyn else None)

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

    def num_parameters(self) -> int:
        return self.params.num_parameters()


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
