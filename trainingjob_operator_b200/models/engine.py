"""What the GPT-2 and BERT training engines share: buffers, kernel-path choice, GEMM and attention front-ends, backward
driver and optimizer.

``TransformerEngine`` owns a model's flat parameters (``flat_params.FlatParams``), the per-layer activation buffers,
the gradient scratch both models use, and the state of the weight-gradient side stream.  The models subclass it with
their parameter specs, their own buffers, ``forward`` and the backward segments ``_bwd_head`` / ``_bwd_layer`` /
``_bwd_tail``.
"""
from __future__ import annotations

import os
from typing import Dict, List, Tuple

import torch
import torch.nn.functional as TF

from .flat_params import FlatParams, ParamSpec


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


# widths at which the engines run fused_ops.cu's LayerNorm pair; layernorm_wide.cu serves every other multiple of 8
FUSED_LAYERNORM_WIDTHS = (256, 512, 768)


class TransformerEngine:
    """Explicit fwd/bwd/optimizer for a fixed (B, T) micro-batch on one GPU.

    ``doc_mask=True`` trains on packed documents: a step also reads ``doc_start`` (int32 [B*T], the sequence-local index of
    the first token of each token's document) and a token attends only to earlier tokens of its own document.  Only the
    wgmma attention kernels implement that mask, so they are used for the forward and the backward, and an engine they
    cannot serve is refused at construction."""

    def __init__(self, cfg, specs: List[ParamSpec], batch_size: int, seq_len: int, device, seed: int, gemm_backend: str,
                 causal: bool, doc_mask: bool):
        from ..ops import functional as F

        assert seq_len <= cfg.block_size
        self.F = F
        self.cfg = cfg
        self.B, self.T = batch_size, seq_len
        self.M = batch_size * seq_len
        self.dev = torch.device(device)
        self.backend = gemm_backend
        self.causal = causal
        self.doc_mask = bool(doc_mask)
        self._choose_kernel_paths()
        self._attn_delta = None
        self._dq_acc = None
        self._philox = torch.zeros((), dtype=torch.int64, device=device)
        self.params = FlatParams(specs, self.dev, seed=seed)
        C, M, Vp = cfg.n_embd, self.M, cfg.padded_vocab
        with torch.no_grad():
            self.params.w32("wte")[cfg.vocab_size:].zero_()
            self.params.refresh_compute_copy()
        bf = dict(device=self.dev, dtype=torch.bfloat16)
        f32 = dict(device=self.dev, dtype=torch.float32)
        self.tok = torch.zeros(M, dtype=torch.int64, device=self.dev)
        self.tgt = torch.zeros(M, dtype=torch.int64, device=self.dev)
        self.doc_start = torch.zeros(M, dtype=torch.int32, device=self.dev) if self.doc_mask else None
        self.layers = [_LayerBufs(M, C, self.dev) for _ in range(cfg.n_layer)]
        self.logits = torch.empty(M, Vp, **bf)
        self.losses = torch.empty(M, **f32)
        self.loss = torch.zeros(1, **f32)
        # backward scratch
        self.d_fc = torch.empty(M, 4 * C, **bf)
        self.d_qkv = torch.empty(M, 3 * C, **bf)
        self.d_att = torch.empty(M, C, **bf)
        # optimizer scalars
        self.sumsq = torch.zeros(1, **f32)
        self.dyn = torch.zeros(4, **f32)
        self._dyn_host = torch.zeros(4, dtype=torch.float32).pin_memory() if self.dev.type == "cuda" else None
        self._wgrad_done = None
        self.segment_join = False     # True: every backward segment joins the side stream (segments are separate graphs)
        self.grad_hook = None  # called as hook(name_of_bucket) when a gradient bucket is complete
        self.split_k: Dict[Tuple[int, int], int] = {}
        # backward GEMMs may leave a few SMs to the gradient all-reduce kernels that run next to them (DDP): a
        # persistent grid of exactly #SMs CTAs needs a second wave as soon as a collective holds some SMs
        self.bwd_max_ctas = 0

    def _choose_kernel_paths(self) -> None:
        """Read the kernel-path switches of docs/ENVIRONMENT.md and settle which kernels this engine launches."""
        if self.backend not in ("wgmma", "cublas"):
            raise ValueError(f"gemm_backend must be 'wgmma' or 'cublas', not {self.backend!r}")
        cfg, T = self.cfg, self.T
        head_dim = cfg.n_embd // cfg.n_head
        # LayerNorm by width: fused_ops.cu's pair where it runs fastest (GPT-2 small, BERT-base); layernorm_wide.cu's
        # for the widths that pair refuses (GPT-2 large 1280, XL 1600) and for 1024 (GPT-2 medium), where the fused
        # backward spills and the wide pair measured faster (docs/gpt2_sizes_h100_700w.json)
        C = cfg.n_embd
        if C in FUSED_LAYERNORM_WIDTHS:
            self.ln_impl = "fused"
        elif C % 8 == 0 and 8 <= C <= self.F.LAYERNORM_WIDE_MAX_C:
            self.ln_impl = "wide"
        else:
            raise ValueError(f"no LayerNorm kernel serves n_embd={C}: the widths served are multiples of 8 up to "
                             f"{self.F.LAYERNORM_WIDE_MAX_C}")
        if self.doc_mask:
            why = [w for bad, w in ((not self.causal, "it needs causal attention"),
                                    (T % 128, f"the sequence length {T} is not a multiple of 128"),
                                    (head_dim != 64, f"the head dim {head_dim} is not 64"),
                                    (self.backend != "wgmma", f"gemm_backend is {self.backend!r}, not 'wgmma'")) if bad]
            if why:
                raise ValueError("document-masked attention runs on the wgmma attention kernels only, which cannot serve "
                                 "this engine: " + "; ".join(why))
            self.attn_impl = self.attn_bwd_impl = "wgmma"
        else:
            # attention forward: "cudnn" (PyTorch SDPA -> cuDNN flash kernel) or "wgmma" (ops/csrc/attention_wgmma.cu)
            self.attn_impl = os.environ.get("AITJ_ATTN", "cudnn")
            if self.attn_impl == "wgmma" and (T % 128 or head_dim != 64 or self.backend != "wgmma"):
                self.attn_impl = "cudnn"
            # attention backward: "wgmma" (ops/csrc/attention_bwd_wgmma.cu: dq/dk/dv written straight into the packed
            # d_qkv) needs our forward's log-sum-exp, so it implies the wgmma forward; "cudnn" = library kernel + gather
            self.attn_bwd_impl = os.environ.get("AITJ_ATTN_BWD", "cudnn") if self.attn_impl == "wgmma" else "cudnn"
        # 2-CTA cluster GEMM: two 128x256 tiles sharing the B tile by TMA multicast (AITJ_GEMM_PAIR=0: single CTAs)
        self.pair = os.environ.get("AITJ_GEMM_PAIR", "1") != "0"
        # per-GEMM kernel choice measured in the step (tools/gemm_cfg_sweep.py): "kind:NxK=block_n[/split_k]" entries,
        # block_n 512 = 2-CTA cluster, 256 / 128 = 1-CTA tiles
        self.gemm_cfg: Dict[str, Tuple[int, int]] = {}
        for item in filter(None, os.environ.get("AITJ_GEMM_CFG", "").split(",")):
            k, v = item.split("=")
            bn, _, sk = v.partition("/")
            self.gemm_cfg[k.strip()] = (int(bn), int(sk or 0))
        # weight-gradient GEMMs on a side stream (AITJ_WGRAD_STREAM=0: in line); see _wgrad
        self.wgrad_stream = torch.cuda.Stream() if (self.dev.type == "cuda" and self.backend == "wgmma" and
                                                    os.environ.get("AITJ_WGRAD_STREAM", "0") != "0") else None

    # ------------------------------------------------------------------ LayerNorm front-ends
    def layernorm_fwd(self, x, gamma, beta, y, mean, rstd):
        """y = LayerNorm(x), with the per-row mean and rstd, on the kernel ``_choose_kernel_paths`` chose."""
        fn = self.F.layernorm_fwd if self.ln_impl == "fused" else self.F.layernorm_wide_fwd
        return fn(x, gamma, beta, y, mean, rstd)

    def layernorm_bwd(self, dy, x, gamma, mean, rstd, dx, dgamma, dbeta, dres=None, dxsum=None):
        """dx = LN'(dy) (+ dres); dgamma, dbeta and dxsum (the previous linear's bias gradient) accumulate."""
        fn = self.F.layernorm_bwd if self.ln_impl == "fused" else self.F.layernorm_wide_bwd
        return fn(dy, x, gamma, mean, rstd, dx, dgamma, dbeta, dres=dres, dxsum=dxsum)

    # ------------------------------------------------------------------ GEMM front-ends
    def _linear(self, x, w, out, bias=None, residual=None, gelu=False, aux=None, block_n=None):
        """out = x @ w^T (+ bias) (GELU, pre-activation to aux) (+ residual).  ``block_n``: the wgmma tile, None = the
        engine's choice for this shape."""
        F = self.F
        if self.backend == "wgmma":
            if block_n is None:
                block_n = self._bn(x.shape[0], w.shape[0], f"fwd:{w.shape[0]}x{w.shape[1]}")
            F.gemm(x, w, out, bias=bias, residual=residual, gelu=gelu, save_pre=gelu, aux=aux, block_n=block_n)
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
            fused = colsum is not None and bn == 512
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

    # ------------------------------------------------------------------ attention
    def _doc_mask_arg(self) -> dict:
        """``doc_start`` for the attention entry points.  Without a mask the keyword is left out, so the call also suits
        stand-ins of those entry points that know no document mask, such as the CPU emulation of the tests."""
        return {} if self.doc_start is None else {"doc_start": self.doc_start}

    def _attention_fwd(self, lb: _LayerBufs):
        B, T, H = self.B, self.T, self.cfg.n_head
        D = self.cfg.n_embd // H
        if self.attn_impl == "wgmma":
            # hand-written flash-attention forward (ops/csrc/attention_wgmma.cu): reads the packed qkv in place,
            # writes [B*T, H*D] and the log-sum-exp the backward needs
            if lb.lse is None:
                lb.lse = torch.empty(B, H, T, device=self.dev, dtype=torch.float32)
            self.F.attention_fwd(lb.qkv, lb.att, lb.lse, B, T, H, causal=self.causal, **self._doc_mask_arg())
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

    def _attention_doc_fwd(self, lb: _LayerBufs, doc_start: torch.Tensor):
        """The wgmma attention forward under the document mask ``doc_start``, whatever ``attn_impl`` training uses
        (scoring completions packed as documents).  The log-sum-exp buffer is allocated on first use when training runs
        cuDNN attention."""
        B, T, H = self.B, self.T, self.cfg.n_head
        if lb.lse is None:
            lb.lse = torch.empty(B, H, T, device=self.dev, dtype=torch.float32)
        self.F.attention_fwd(lb.qkv, lb.att, lb.lse, B, T, H, causal=True, doc_start=doc_start)
        lb.att_in = lb.att

    def _attention_bwd(self, lb: _LayerBufs, d_att: torch.Tensor, d_qkv: torch.Tensor, d_bias: torch.Tensor):
        """d_qkv <- SDPA backward; d_bias (the qkv bias gradient) += colsum(d_qkv), fused into the gather."""
        B, T, H = self.B, self.T, self.cfg.n_head
        D = self.cfg.n_embd // H
        if self.attn_bwd_impl == "wgmma":
            if self._dq_acc is None:
                self._attn_delta = torch.empty(B, H, T, device=self.dev, dtype=torch.float32)
                self._dq_acc = torch.zeros(B * T, H * D, device=self.dev, dtype=torch.float32)
            self.F.attention_bwd(lb.qkv, lb.att, d_att, lb.lse, self._attn_delta, self._dq_acc, d_qkv, B, T, H,
                                 causal=self.causal, **self._doc_mask_arg())
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
        self.F.qkv_gather_colsum(dq, dk, dv, d_qkv, d_bias)
        lb.sdpa_ctx = None

    # ------------------------------------------------------------------ loss / backward
    def _loss(self, n: int) -> torch.Tensor:
        """self.loss = sum of the per-token losses / n; leaves dlogits (scaled by 1 / n) in self.logits."""
        self.F.softmax_xent(self.logits, self.tgt, self.losses, self.cfg.vocab_size, 1.0 / n)
        torch.sum(self.losses, dim=0, keepdim=True, out=self.loss)
        self.loss.mul_(1.0 / n)
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

    def num_parameters(self) -> int:
        return self.params.num_parameters()
