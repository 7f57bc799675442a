"""Python entry points of the hand-written sm_90a kernels (ctypes -> libaitj_kernels.so).

Every function launches on ``torch.cuda.current_stream()`` and works on preallocated
tensors, so a whole training step can be captured in one CUDA graph.  There is deliberately
no eager/PyTorch fallback here: on a GPU box a missing library raises.
"""
from __future__ import annotations

import torch

from . import lib

EPI_BIAS = 1
EPI_GELU = 2
EPI_RESIDUAL = 4
EPI_SAVE_PRE = 8
EPI_DGELU = 16
EPI_OUT_F32 = 32
EPI_ACCUM = 64
EPI_MC = 128
EPI_PEER = 16384
EPI_COLSUM = 256   # set by the library when a colsum buffer is given
EPI_XENT = 512     # gemm_xent: per-row cross-entropy partials instead of an output (kernel keyed EPI_XENT | EPI_OUT_F32)

# aitj_gemm_bf16: out, aux or residual is not 16-byte aligned (the epilogue reaches them by TMA)
GEMM_MISALIGNED = -4
# aitj_gemm_bf16: no kernel is compiled for this operand layout and epilogue
GEMM_NO_KERNEL = -7


class RawView:
    """A (pointer, shape, dtype) triple standing in for a tensor: used to aim gradient-producing kernels at the
    NVSwitch *multicast* alias of a symmetric buffer (an address torch has no tensor for)."""

    is_multicast = True

    def __init__(self, ptr: int, shape, dtype, row_stride=None):
        self._ptr = int(ptr)
        self.shape = tuple(shape)
        self.dtype = dtype
        self._rs = row_stride if row_stride is not None else (self.shape[-1] if len(self.shape) > 1 else 1)

    def data_ptr(self) -> int:
        return self._ptr

    def stride(self, i: int) -> int:
        return self._rs if (i == 0 and len(self.shape) > 1) else 1

    def dim(self) -> int:
        return len(self.shape)


class PeerView:
    """A gradient tensor inside the symmetric, owner-sharded buffer (``parallel.symm.ShardedGradState``): kernels are
    given its LOCAL address and add into the copy of the rank that owns each piece."""

    is_peer = True

    def __init__(self, t: torch.Tensor):
        self.t = t
        self.shape = tuple(t.shape)
        self.dtype = t.dtype

    def data_ptr(self) -> int:
        return self.t.data_ptr()

    def stride(self, i: int) -> int:
        return self.t.stride(i)

    def dim(self) -> int:
        return self.t.dim()


def _is_mc(t) -> int:
    """Gradient accumulation mode of a destination: 0 local atomics, 1 NVSwitch multicast, 2 owner's copy (peer)."""
    if getattr(t, "is_peer", False):
        return 2
    return 1 if getattr(t, "is_multicast", False) else 0

_NUM_SMS = None


def num_sms() -> int:
    global _NUM_SMS
    if _NUM_SMS is None:
        _NUM_SMS = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    return _NUM_SMS


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _ptr(t):
    return None if t is None else t.data_ptr()


def gemm(a, b, out, *, a_mn=False, b_mn=False, bias=None, residual=None, aux=None, gelu=False, dgelu=False,
         save_pre=False, accumulate=False, split_k=1, block_n=0, max_ctas=0, colsum=None):
    """out[M,N] (+)= opA[M,K] @ opB[N,K]^T on wgmma tensor cores (bf16 in, fp32 accumulate).

    a_mn=False: ``a`` is [M,K]; a_mn=True: ``a`` is [K,M] (its transpose is used).
    b_mn=False: ``b`` is [N,K]; b_mn=True: ``b`` is [K,N].
    ``out`` bf16 -> plain store; fp32 -> store, or red.add when ``accumulate`` (needed for split_k>1).
    Epilogue: +bias[N] -> (aux<-pre) -> gelu -> *gelu'(aux) -> +residual[M,N].
    ``block_n``: 128 / 256 = tile width, 0 = auto, 512 / 1024 = 128x256 tiles in clusters of 2 / 4 CTAs that share the
    B tile by TMA multicast.
    ``colsum`` (fp32[N], bf16 output only): += column sums of the stored output.
    """
    assert a.dtype == torch.bfloat16 and b.dtype == torch.bfloat16
    assert a.dim() == 2 and b.dim() == 2 and a.stride(1) == 1 and b.stride(1) == 1 and out.stride(1) == 1
    if a_mn:
        K, M = a.shape
    else:
        M, K = a.shape
    if b_mn:
        Kb, N = b.shape
    else:
        N, Kb = b.shape
    assert K == Kb, (a.shape, b.shape, a_mn, b_mn)
    assert out.shape[0] == M and out.shape[1] == N, (out.shape, M, N)
    flags = gemm_epilogue(out, bias=bias, residual=residual, aux=aux, gelu=gelu, dgelu=dgelu, save_pre=save_pre,
                          accumulate=accumulate, colsum=colsum)
    if colsum is not None:
        lib.load().aitj_gemm_set_colsum(colsum.data_ptr())
    try:
        lib.call("aitj_gemm_bf16", a.data_ptr(), b.data_ptr(), out.data_ptr(), M, N, K, a.stride(0), b.stride(0),
                 out.stride(0), int(a_mn), int(b_mn), _ptr(bias), _ptr(residual), _ptr(aux), flags & ~EPI_COLSUM,
                 int(split_k), int(block_n), int(max_ctas), _stream())
    except lib.KernelError as e:
        if e.code != GEMM_NO_KERNEL:
            raise
        raise lib.KernelError(f"no wgmma GEMM kernel is compiled for a_mn={int(a_mn)} b_mn={int(b_mn)} with epilogue "
                              f"{epilogue_name(flags)}; add the pair to kGemmKernels in gemm_wgmma.cu",
                              e.code) from None
    return out


def epilogue_name(flags: int) -> str:
    names = [n for n, bit in (("BIAS", EPI_BIAS), ("GELU", EPI_GELU), ("RESIDUAL", EPI_RESIDUAL),
                              ("SAVE_PRE", EPI_SAVE_PRE), ("DGELU", EPI_DGELU), ("OUT_F32", EPI_OUT_F32),
                              ("ACCUM", EPI_ACCUM), ("MC", EPI_MC), ("PEER", EPI_PEER), ("COLSUM", EPI_COLSUM),
                              ("XENT", EPI_XENT))
             if flags & bit]
    return "|".join(names) or "none"


def xent_blocks(n: int) -> int:
    """Column blocks of ``gemm_xent``'s partials for a product with ``n`` columns."""
    return (n + 127) // 128


def gemm_xent(x, w, target, vocab, part, tgt_logit, block_n=0):
    """Cross-entropy partials of the logits x[M,K] @ w[N,K]^T, which are never written out: for every row r with
    target[r] >= 0 (int64 [M]), part[r, b] <- (max, sum of exp(z - max)) over the columns z < ``vocab`` of 128-column
    block b (fp32 [M, xent_blocks(N), 2]) and tgt_logit[r] <- the logit of column target[r] (fp32 [M]), from the fp32
    accumulators.  ``xent_finish`` turns them into per-row losses.  ``block_n`` as for ``gemm``."""
    assert x.dtype == torch.bfloat16 and w.dtype == torch.bfloat16 and x.dim() == 2 and w.dim() == 2
    assert x.stride(1) == 1 and w.stride(1) == 1
    M, K = x.shape
    N, Kw = w.shape
    assert K == Kw, (x.shape, w.shape)
    assert 0 < vocab <= N, (vocab, N)
    assert target.dtype == torch.int64 and target.numel() == M and target.is_contiguous()
    assert part.dtype == torch.float32 and tuple(part.shape) == (M, xent_blocks(N), 2) and part.is_contiguous()
    assert tgt_logit.dtype == torch.float32 and tgt_logit.numel() == M
    lib.load().aitj_gemm_set_xent(target.data_ptr(), part.data_ptr(), tgt_logit.data_ptr(), int(vocab))
    lib.call("aitj_gemm_bf16", x.data_ptr(), w.data_ptr(), None, M, N, K, x.stride(0), w.stride(0), 0, 0, 0, None,
             None, None, EPI_XENT, 1, int(block_n), 0, _stream())


def xent_finish(part, tgt_logit, target, loss, acc):
    """loss[r] <- log-sum-exp of row r's ``gemm_xent`` partials - tgt_logit[r] (0 where target[r] < 0); acc (fp64 [2])
    += (sum of the losses, rows with a target)."""
    M, nblk = part.shape[0], part.shape[1]
    assert acc.dtype == torch.float64 and acc.numel() == 2 and loss.dtype == torch.float32 and loss.numel() == M
    lib.call("aitj_xent_finish", part.data_ptr(), tgt_logit.data_ptr(), target.data_ptr(), loss.data_ptr(),
             acc.data_ptr(), M, nblk, _stream())


def gemm_epilogue(out, *, bias=None, residual=None, aux=None, gelu=False, dgelu=False, save_pre=False,
                  accumulate=False, colsum=None) -> int:
    """The EPI_* bits of a ``gemm`` call with these arguments; EPI_COLSUM marks a colsum buffer."""
    flags = 0
    if bias is not None:
        flags |= EPI_BIAS
    if gelu:
        flags |= EPI_GELU
    if residual is not None:
        flags |= EPI_RESIDUAL
        assert residual.stride(0) == out.stride(0)
    if save_pre:
        flags |= EPI_SAVE_PRE
    if dgelu:
        flags |= EPI_DGELU
    if save_pre or dgelu:
        assert aux is not None and aux.stride(0) == out.stride(0)
    if out.dtype == torch.float32:
        flags |= EPI_ACCUM if accumulate else EPI_OUT_F32
        if _is_mc(out) == 1:
            assert accumulate, "multicast outputs are reduce-only"
            flags |= EPI_MC
        elif _is_mc(out) == 2:
            assert accumulate, "owner-sharded outputs are reduce-only"
            flags |= EPI_PEER
    else:
        assert out.dtype == torch.bfloat16 and not accumulate
    if colsum is not None:
        assert colsum.dtype == torch.float32 and colsum.numel() == out.shape[1] and out.dtype == torch.bfloat16
        flags |= EPI_COLSUM
    return flags


def auto_split_k(M: int, N: int, K: int, block_n: int = 0, pair: bool = False) -> int:
    """Split-K factor for a weight-gradient shaped GEMM (small MxN, huge K): the split that best fills whole
    waves of SMs (or SM pairs), keeping at least 16 k-blocks per split; ties go to the smaller split."""
    if pair:
        tiles = ((M + 255) // 256) * ((N + 255) // 256)
        slots = max(1, num_sms() // 2)
    else:
        bn = block_n or (256 if N > 128 else 128)
        tiles = ((M + 127) // 128) * ((N + bn - 1) // bn)
        slots = num_sms()
    if tiles >= slots:
        return 1
    kb = (K + 63) // 64
    best, best_eff = 1, 0.0
    for s in range(1, 33):
        if s > 1 and kb // s < 16:
            break
        work = tiles * s
        eff = work / (((work + slots - 1) // slots) * slots)
        if eff > best_eff + 0.02:
            best, best_eff = s, eff
    return best


def layernorm_fwd(x, gamma, beta, y, mean, rstd, eps=1e-5):
    M, C = x.shape
    lib.call("aitj_layernorm_fwd", x.data_ptr(), gamma.data_ptr(), beta.data_ptr(), y.data_ptr(), mean.data_ptr(),
             rstd.data_ptr(), M, C, float(eps), _stream())
    return y


def layernorm_bwd(dy, x, gamma, mean, rstd, dx, dgamma, dbeta, dres=None, dxsum=None):
    """dx = LN'(dy) (+ dres); dgamma/dbeta (fp32) are accumulated; dxsum (fp32[C], optional) += colsum(dx),
    which is the bias gradient of the linear layer that produced this LayerNorm's input."""
    M, C = x.shape
    lib.call("aitj_layernorm_bwd", dy.data_ptr(), x.data_ptr(), gamma.data_ptr(), mean.data_ptr(), rstd.data_ptr(),
             _ptr(dres), dx.data_ptr(), dgamma.data_ptr(), dbeta.data_ptr(), _ptr(dxsum), M, C, _is_mc(dgamma),
             _stream())
    return dx


# ------------------------------------------------------------------------------------ wide LayerNorm (layernorm_wide.cu)
# For the widths the pair above refuses, such as GPT-2 large (1280) and XL (1600): any C that is a multiple of 8, up to
# LAYERNORM_WIDE_MAX_C.  Like the decode entry points, the library refuses nothing; every argument is checked here.
LAYERNORM_WIDE_MAX_C = 2048


def _check_rows(t, name: str, M: int, C: int) -> None:
    _tensor(t, name, torch.bfloat16, 2, 16)
    _need(tuple(t.shape) == (M, C), f"{name} must be [{M}, {C}], not {tuple(t.shape)}")


def _check_wide_input(x, gamma, mean, rstd):
    _tensor(x, "x", torch.bfloat16, 2, 16)
    M, C = x.shape
    _need(C % 8 == 0 and 8 <= C <= LAYERNORM_WIDE_MAX_C,
          f"the wide LayerNorm needs a width that is a multiple of 8 in [8, {LAYERNORM_WIDE_MAX_C}], not {C}")
    _tensor(gamma, "gamma", torch.bfloat16, 1, 8)
    _need(gamma.numel() == C, f"gamma must hold {C} elements, not {gamma.numel()}")
    for t, name in ((mean, "mean"), (rstd, "rstd")):
        _tensor(t, name, torch.float32, 1)
        _need(t.numel() == M, f"{name} must hold {M} elements, not {t.numel()}")
    return M, C


def check_layernorm_wide_fwd(x, gamma, beta, y, mean, rstd, eps=1e-5):
    """(M, C) of a valid ``layernorm_wide_fwd`` call; ValueError otherwise."""
    M, C = _check_wide_input(x, gamma, mean, rstd)
    _tensor(beta, "beta", torch.bfloat16, 1, 8)
    _need(beta.numel() == C, f"beta must hold {C} elements, not {beta.numel()}")
    _check_rows(y, "y", M, C)
    return M, C


def layernorm_wide_fwd(x, gamma, beta, y, mean, rstd, eps=1e-5):
    """``layernorm_fwd`` for any width that is a multiple of 8 up to ``LAYERNORM_WIDE_MAX_C``: y (bf16), and the fp32
    per-row mean and rstd the backward reads."""
    M, C = check_layernorm_wide_fwd(x, gamma, beta, y, mean, rstd, eps)
    lib.call("aitj_layernorm_wide_fwd", x.data_ptr(), gamma.data_ptr(), beta.data_ptr(), y.data_ptr(), mean.data_ptr(),
             rstd.data_ptr(), M, C, float(eps), _stream())
    return y


def check_layernorm_wide_bwd(dy, x, gamma, mean, rstd, dx, dgamma, dbeta, dres=None, dxsum=None):
    """(M, C) of a valid ``layernorm_wide_bwd`` call; ValueError otherwise."""
    M, C = _check_wide_input(x, gamma, mean, rstd)
    _check_rows(dy, "dy", M, C)
    _check_rows(dx, "dx", M, C)
    if dres is not None:
        _check_rows(dres, "dres", M, C)
    mode = _is_mc(dgamma)
    for t, name in ((dgamma, "dgamma"), (dbeta, "dbeta"), (dxsum, "dxsum")):
        if t is None and name == "dxsum":
            continue
        _need(t is not None and t.dtype == torch.float32 and tuple(t.shape) == (C,),
              f"{name} must be an fp32 gradient of shape ({C},)")
        _need(not isinstance(t, torch.Tensor) or t.is_contiguous(), f"{name} must be contiguous")
        _need(t.data_ptr() % 4 == 0, f"{name} must be 4-byte aligned")
        _need(_is_mc(t) == mode, "dgamma, dbeta and dxsum must all be local, all multicast or all owner-sharded")
    return M, C


def layernorm_wide_bwd(dy, x, gamma, mean, rstd, dx, dgamma, dbeta, dres=None, dxsum=None):
    """``layernorm_bwd`` for the widths of ``layernorm_wide_fwd``, with the same fusions: dx = LN'(dy) (+ dres) in bf16;
    dgamma, dbeta and dxsum (optional: colsum(dx), the bias gradient of the linear layer that produced x) are added to
    fp32 gradients, local, multicast or owner-sharded."""
    M, C = check_layernorm_wide_bwd(dy, x, gamma, mean, rstd, dx, dgamma, dbeta, dres, dxsum)
    lib.call("aitj_layernorm_wide_bwd", dy.data_ptr(), x.data_ptr(), gamma.data_ptr(), mean.data_ptr(),
             rstd.data_ptr(), _ptr(dres), dx.data_ptr(), dgamma.data_ptr(), dbeta.data_ptr(), _ptr(dxsum), M, C,
             _is_mc(dgamma), _stream())
    return dx


def embedding_fwd(tok, wte, wpe, out, T):
    M, C = out.shape
    lib.call("aitj_embedding_fwd", tok.data_ptr(), wte.data_ptr(), _ptr(wpe), out.data_ptr(), M, T, C, _stream())
    return out


def embedding_bwd(tok, dx, dwte, dwpe, T):
    M, C = dx.shape
    lib.call("aitj_embedding_bwd", tok.data_ptr(), dx.data_ptr(), dwte.data_ptr(), _ptr(dwpe), M, T, C, _is_mc(dwte),
             _stream())


def embedding3_fwd(tok, typ, wte, wpe, wtt, out, T):
    """out = wte[tok] + wpe[position] + wtt[typ] (BERT: word + position + token-type embeddings)."""
    M, C = out.shape
    lib.call("aitj_embedding3_fwd", tok.data_ptr(), typ.data_ptr(), wte.data_ptr(), wpe.data_ptr(), wtt.data_ptr(),
             out.data_ptr(), M, T, C, _stream())
    return out


def embedding3_bwd(tok, typ, dx, dwte, dwpe, dwtt, T):
    M, C = dx.shape
    lib.call("aitj_embedding3_bwd", tok.data_ptr(), typ.data_ptr(), dx.data_ptr(), dwte.data_ptr(), dwpe.data_ptr(),
             dwtt.data_ptr(), M, T, C, _is_mc(dwte), _stream())


def softmax_xent(logits, target, loss, V, gscale):
    """In place: logits[M,Vp] <- dlogits = (softmax - onehot) * gscale; loss[M] <- per-row NLL."""
    M, Vp = logits.shape
    lib.call("aitj_softmax_xent", logits.data_ptr(), target.data_ptr(), loss.data_ptr(), M, V, Vp, float(gscale),
             _stream())


def colsum(dy, db):
    M, N = dy.shape
    lib.call("aitj_colsum", dy.data_ptr(), db.data_ptr(), M, N, _is_mc(db), _stream())


def _check_doc_start(doc_start, B, T, causal):
    """``doc_start``: int32 [B*T], the sequence-local index of the first token of the document holding each token; query
    q then sees key k iff doc_start[q] <= k <= q.  Only a causal attention takes one."""
    if doc_start is None:
        return None
    if not causal:
        raise ValueError("a document mask needs causal attention")
    if doc_start.dtype != torch.int32 or not doc_start.is_contiguous() or doc_start.numel() != B * T:
        raise ValueError(f"doc_start must be a contiguous int32 tensor of {B * T} elements, got "
                         f"{doc_start.dtype} {tuple(doc_start.shape)}")
    if doc_start.data_ptr() % 8:
        raise ValueError("doc_start must be 8-byte aligned (the kernels read it in pairs)")
    return doc_start.data_ptr()


def attention_fwd(qkv, out, lse, B, T, H, causal=True, scale=0.0, doc_start=None):
    """Flash attention forward on wgmma (head dim 64): qkv bf16 [B*T, 3*H*64] packed q|k|v -> out bf16 [B*T, H*64],
    lse fp32 [B, H, T] (natural-log sum-exp of the scaled scores).  T % 128 == 0.  ``doc_start`` (int32 [B*T], causal
    only): document mask of packed sequences, see ``_check_doc_start``."""
    assert qkv.dtype == torch.bfloat16 and out.dtype == torch.bfloat16 and lse.dtype == torch.float32
    assert qkv.is_contiguous() and out.is_contiguous() and lse.is_contiguous()
    assert qkv.shape == (B * T, 3 * H * 64) and out.shape == (B * T, H * 64) and lse.numel() == B * H * T
    ds = _check_doc_start(doc_start, B, T, causal)
    lib.call("aitj_attn_fwd", qkv.data_ptr(), out.data_ptr(), lse.data_ptr(), ds, B, T, H, int(causal), float(scale),
             _stream())
    return out


def attention_bwd(qkv, out, d_out, lse, delta, dq_acc, d_qkv, B, T, H, causal=True, scale=0.0, doc_start=None):
    """Flash attention backward on wgmma (head dim 64).  qkv / d_qkv bf16 [B*T, 3*H*64] (d_qkv receives dq | dk | dv in
    place), out / d_out bf16 [B*T, H*64], lse fp32 [B,H,T] from ``attention_fwd``; delta fp32 [B,H,T] and dq_acc fp32
    [B*T, H*64] are scratch -- dq_acc must be zero on entry and is zero again on exit.  ``doc_start``: the document mask
    the forward was given."""
    assert qkv.dtype == torch.bfloat16 and d_qkv.dtype == torch.bfloat16 and dq_acc.dtype == torch.float32
    assert qkv.is_contiguous() and out.is_contiguous() and d_out.is_contiguous() and d_qkv.is_contiguous()
    assert qkv.shape == (B * T, 3 * H * 64) and d_qkv.shape == qkv.shape and out.shape == (B * T, H * 64)
    assert d_out.shape == out.shape and dq_acc.shape == out.shape and lse.numel() == B * H * T == delta.numel()
    ds = _check_doc_start(doc_start, B, T, causal)
    lib.call("aitj_attn_bwd", qkv.data_ptr(), out.data_ptr(), d_out.data_ptr(), lse.data_ptr(), delta.data_ptr(),
             dq_acc.data_ptr(), d_qkv.data_ptr(), ds, B, T, H, int(causal), float(scale), _stream())
    lib.LAUNCHES += 2          # delta + dq_finish ride along with the main kernel
    return d_qkv


def qkv_gather_colsum(dq, dk, dv, d_qkv, db):
    """d_qkv[B*T, 3*H*D] <- (dq, dk, dv), each logically [B,H,T,D] with any B/H/T strides; db[3*H*D] += colsum."""
    import ctypes

    B, H, T, D = dq.shape
    st = []
    for t in (dq, dk, dv):
        if t.stride(3) != 1 or tuple(t.shape) != (B, H, T, D):
            raise ValueError("qkv_gather_colsum: need [B,H,T,D] tensors with unit D stride")
        st += [t.stride(0), t.stride(1), t.stride(2)]
    arr = (ctypes.c_longlong * 9)(*st)
    lib.call("aitj_qkv_gather_colsum", dq.data_ptr(), dk.data_ptr(), dv.data_ptr(), ctypes.addressof(arr),
             d_qkv.data_ptr(), db.data_ptr(), B, T, H, D, _is_mc(db), _stream())


def sumsq(g, out):
    lib.call("aitj_sumsq", g.data_ptr(), g.numel(), out.data_ptr(), _stream())


def adamw(p, g, m, v, p16, wd_mask, *, lr, beta1=0.9, beta2=0.95, eps=1e-8, weight_decay=0.1, step=1, sumsq_buf=None,
          max_norm=0.0, grad_div=1.0, zero_grad=True, dyn=None, sumsq_n=1, p16_multicast=False):
    """One sweep: AdamW on fp32 master state + bf16 compute copy refresh + grad zeroing.
    ``dyn`` (device float[3] = lr, 1-beta1^t, 1-beta2^t) overrides lr/step for CUDA-graph replay.
    ``sumsq_n`` > 1: ``sumsq_buf`` holds that many partial square sums (one per rank).  ``p16_multicast``: ``p16`` is an
    int -- the NVSwitch multicast address of this range of the bf16 copy -- and the sweep stores into every rank's copy."""
    if sumsq_n != 1 or p16_multicast:
        lib.load().aitj_adamw_set_shard(int(sumsq_n), int(bool(p16_multicast)))
    p16_ptr = int(p16) if p16_multicast else p16.data_ptr()
    lib.call("aitj_adamw", p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), p16_ptr, wd_mask.data_ptr(),
             _ptr(sumsq_buf), _ptr(dyn), p.numel(), float(lr), float(beta1), float(beta2), float(eps), float(weight_decay),
             int(step), float(max_norm), float(grad_div), int(bool(zero_grad)), _stream())


def mc_push(dst_mc_ptr: int, src, n: int):
    """dst_mc[0:n] (+)= src[0:n] through the NVSwitch multicast alias; src is cleared."""
    lib.call("aitj_mc_push", int(dst_mc_ptr), src.data_ptr(), int(n), _stream())


def peer_push(dst_local, src):
    """Owner-sharded mode: dst_local[i] (in the owner's copy) += src[i]; src is cleared."""
    lib.call("aitj_peer_push", dst_local.data_ptr(), src.data_ptr(), int(src.numel()), _stream())


def norm_share(parts_mc_ptr: int, mine, rank: int):
    """parts[rank] <- mine[0] in every rank's copy (multicast store)."""
    lib.call("aitj_norm_share", int(parts_mc_ptr), mine.data_ptr(), int(rank), _stream())


def cast_f32_bf16(src, dst):
    lib.call("aitj_cast_f32_bf16", src.data_ptr(), dst.data_ptr(), src.numel(), _stream())


def gelu_fwd(x, y):
    lib.call("aitj_gelu_fwd", x.data_ptr(), y.data_ptr(), x.numel(), _stream())


def gelu_bwd(x, dy, dx):
    lib.call("aitj_gelu_bwd", x.data_ptr(), dy.data_ptr(), dx.data_ptr(), x.numel(), _stream())


# ------------------------------------------------------------------------------------ decoding (ops/csrc/decode.cu)
# The decode entry points refuse nothing themselves: every argument is checked here, before the library is called.
# ``check_*`` are the checks alone, so that stand-ins of these entry points can apply the same ones.
DECODE_CHUNK = 64            # cache positions per attention_decode CTA
SAMPLE_MAX_VOCAB = 102400    # sample_tokens stages a bf16 row of the vocabulary in shared memory (200 KB)


def _need(ok: bool, msg: str) -> None:
    if not ok:
        raise ValueError(msg)


def _tensor(t, name: str, dtype, ndim: int = None, align: int = 0) -> None:
    _need(isinstance(t, torch.Tensor), f"{name} must be a tensor")
    _need(t.dtype == dtype, f"{name} must be {dtype}, not {t.dtype}")
    _need(t.is_contiguous(), f"{name} must be contiguous")
    _need(ndim is None or t.dim() == ndim, f"{name} must have {ndim} dimensions, not {t.dim()}")
    _need(not align or t.data_ptr() % align == 0, f"{name} must be {align}-byte aligned")


def _check_pos(pos, n: int) -> None:
    _tensor(pos, "pos", torch.int32)
    _need(pos.numel() >= n, f"pos must hold at least {n} int32 elements")


def decode_partials(S: int, H: int, Tmax: int) -> int:
    """fp32 elements of ``attention_decode``'s scratch: (max, sum, 64 accumulators) per (sequence, head, key chunk)."""
    return S * H * (-(-Tmax // DECODE_CHUNK)) * (64 + 2)


def check_attention_decode(qkv, cache, pos, out, part, H: int):
    """(S, Tmax) of a valid ``attention_decode`` call; ValueError otherwise."""
    _tensor(qkv, "qkv", torch.bfloat16, 2, 16)
    S = qkv.shape[0]
    _need(S >= 1, "attention_decode needs S >= 1 sequences")
    _need(H >= 1 and qkv.shape[1] == 3 * H * 64, f"qkv has {qkv.shape[1]} columns: H * 64 == C needs 3 * {H} * 64")
    _tensor(cache, "cache", torch.bfloat16, 5, 16)
    _need(cache.shape[0] == S and cache.shape[2:] == (2, H, 64),
          f"cache must be [S={S}, Tmax, 2, H={H}, 64], not {tuple(cache.shape)}")
    Tmax = cache.shape[1]
    _need(Tmax >= 1, "cache must hold at least one position")
    _tensor(out, "out", torch.bfloat16, 2, 16)
    _need(tuple(out.shape) == (S, H * 64), f"out must be [{S}, {H * 64}], not {tuple(out.shape)}")
    _tensor(part, "part", torch.float32)
    _need(part.numel() >= decode_partials(S, H, Tmax), f"part must hold {decode_partials(S, H, Tmax)} fp32 elements")
    _check_pos(pos, 1)
    return S, Tmax


def attention_decode(qkv, cache, pos, out, part, H: int):
    """One decode step of one layer for S sequences at the shared position pos[0] (device int32 < Tmax): the new k and v
    (columns C..3C of qkv bf16 [S, 3C], head dim 64) are written into cache bf16 [S, Tmax, 2, H, 64] at pos[0], and q
    attends over positions [0, pos[0]] -> out bf16 [S, C].  ``part``: fp32 scratch of ``decode_partials`` elements."""
    S, Tmax = check_attention_decode(qkv, cache, pos, out, part, H)
    lib.call("aitj_attention_decode", qkv.data_ptr(), cache.data_ptr(), pos.data_ptr(), out.data_ptr(), part.data_ptr(),
             S, H, Tmax, _stream())
    lib.LAUNCHES += 1          # the merge of the key chunks rides along with the main kernel
    return out


def check_embedding_decode(tok, wte, wpe, pos, out) -> int:
    """S of a valid ``embedding_decode`` call; ValueError otherwise."""
    _tensor(tok, "tok", torch.int64, 1)
    S = tok.numel()
    _need(S >= 1, "embedding_decode needs S >= 1 sequences")
    _tensor(wte, "wte", torch.bfloat16, 2, 16)
    _tensor(wpe, "wpe", torch.bfloat16, 2, 16)
    C = wte.shape[1]
    _need(C % 8 == 0 and wpe.shape[1] == C, f"wte and wpe need the same width, a multiple of 8: {C}, {wpe.shape[1]}")
    _tensor(out, "out", torch.bfloat16, 2, 16)
    _need(tuple(out.shape) == (S, C), f"out must be [{S}, {C}], not {tuple(out.shape)}")
    _check_pos(pos, 1)
    return S


def embedding_decode(tok, wte, wpe, pos, out):
    """out[s] = wte[tok[s]] + wpe[pos[0]] (tok int64 [S], pos device int32)."""
    S = check_embedding_decode(tok, wte, wpe, pos, out)
    lib.call("aitj_embedding_decode", tok.data_ptr(), wte.data_ptr(), wpe.data_ptr(), pos.data_ptr(), out.data_ptr(),
             S, wte.shape[1], _stream())
    return out


def check_sample_tokens(logits, vocab, tok, out_tokens, prompt, prompt_len, pos, temperature, top_k, seed,
                        first_seq=0) -> int:
    """S of a valid ``sample_tokens`` call; ValueError otherwise."""
    _need(isinstance(logits, torch.Tensor) and logits.dtype == torch.bfloat16 and logits.dim() == 2,
          "logits must be a 2-D bf16 tensor")
    _need(logits.stride(1) == 1 and logits.stride(0) >= logits.shape[1], "logits rows must be contiguous")
    S = logits.shape[0]
    _need(S >= 1, "sample_tokens needs S >= 1 sequences")
    _need(1 <= vocab <= logits.shape[1], f"vocab {vocab} must be in [1, {logits.shape[1]}] (the logits' columns)")
    _need(vocab <= SAMPLE_MAX_VOCAB, f"vocab {vocab} exceeds {SAMPLE_MAX_VOCAB}: a row must fit in shared memory")
    _tensor(tok, "tok", torch.int64, 1)
    _need(tok.numel() == S, f"tok must hold {S} tokens, not {tok.numel()}")
    _tensor(out_tokens, "out_tokens", torch.int64, 2)
    _need(out_tokens.shape[0] == S, f"out_tokens must have {S} rows, not {out_tokens.shape[0]}")
    _tensor(prompt, "prompt", torch.int64, 2)
    _need(prompt.shape[0] == S, f"prompt must have {S} rows, not {prompt.shape[0]}")
    _need(1 <= prompt_len <= prompt.shape[1], f"prompt_len {prompt_len} must be in [1, {prompt.shape[1]}]")
    _check_pos(pos, 2)
    _need(temperature >= 0 and temperature < float("inf"), f"temperature must be finite and >= 0, not {temperature}")
    _need(0 <= top_k <= vocab, f"top_k must be in [0, vocab={vocab}], not {top_k}")
    _need(0 <= seed < 1 << 63, f"seed must be in [0, 2^63), not {seed}")
    _need(0 <= first_seq and first_seq + S <= 1 << 31, f"first_seq {first_seq} out of range")
    return S


def sample_tokens(logits, vocab, tok, out_tokens, prompt, prompt_len, pos, temperature, top_k, seed, first_seq=0):
    """The next token of each sequence from its logits row (bf16 [S, Vp], columns >= ``vocab`` never chosen), at the shared
    position p = pos[0]: the prompt's token prompt[s, p + 1] while p + 1 < prompt_len; else the argmax (lowest index on
    ties) when ``temperature`` is 0 or ``top_k`` is 1; else one draw from softmax(logits / temperature) over the ``top_k``
    largest logits (0 = all; ties with the top_k-th are kept), keyed by a Philox counter of (seed, first_seq + s, p), so
    a sequence's tokens never depend on S or its row.  Writes tok[s] and out_tokens[s, p + 1] (when in range), then moves
    pos[0] to p + 1; pos[1] is the kernel's completion count and must be 0 (it is 0 again afterwards)."""
    S = check_sample_tokens(logits, vocab, tok, out_tokens, prompt, prompt_len, pos, temperature, top_k, seed,
                            first_seq)
    lib.call("aitj_sample_tokens", logits.data_ptr(), logits.stride(0), int(vocab), tok.data_ptr(),
             out_tokens.data_ptr(), out_tokens.shape[1], prompt.data_ptr(), prompt.shape[1], int(prompt_len),
             pos.data_ptr(), float(temperature), int(top_k), int(seed), int(first_seq), S, _stream())
    return tok


# ------------------------------------------------------------------------------------ HellaSwag (ops/csrc/hellaswag.cu)
# Scoring completions packed as documents into rows (runtime/hellaswag.py).  Like the decode entry points, the library
# refuses nothing; every argument is checked here.
CHOICES = 4                  # completions per example


def check_embedding_doc_fwd(tok, wte, wpe, doc_start, out, T: int):
    """(M, C) of a valid ``embedding_doc_fwd`` call; ValueError otherwise."""
    _tensor(tok, "tok", torch.int64, 1)
    M = tok.numel()
    _need(M >= 1, "embedding_doc_fwd needs M >= 1 rows")
    _tensor(wte, "wte", torch.bfloat16, 2, 16)
    _tensor(wpe, "wpe", torch.bfloat16, 2, 16)
    C = wte.shape[1]
    _need(C % 8 == 0 and wpe.shape[1] == C, f"wte and wpe need the same width, a multiple of 8: {C}, {wpe.shape[1]}")
    _need(1 <= T <= wpe.shape[0], f"T {T} must be in [1, {wpe.shape[0]}] (the rows of wpe)")
    _need(M % T == 0, f"M {M} is not a multiple of T {T}")
    _tensor(doc_start, "doc_start", torch.int32, 1, 8)
    _need(doc_start.numel() == M, f"doc_start must hold {M} elements, not {doc_start.numel()}")
    _tensor(out, "out", torch.bfloat16, 2, 16)
    _need(tuple(out.shape) == (M, C), f"out must be [{M}, {C}], not {tuple(out.shape)}")
    return M, C


def embedding_doc_fwd(tok, wte, wpe, doc_start, out, T: int):
    """out[r] = wte[tok[r]] + wpe[(r mod T) - doc_start[r]]: ``embedding_fwd`` with positions counted from the first
    token of each row's document (doc_start int32 [M], as the document-masked attention takes it)."""
    M, C = check_embedding_doc_fwd(tok, wte, wpe, doc_start, out, T)
    lib.call("aitj_embedding_doc_fwd", tok.data_ptr(), wte.data_ptr(), wpe.data_ptr(), doc_start.data_ptr(),
             out.data_ptr(), M, int(T), C, _stream())
    return out


def check_choice_score(loss, spans, labels, mean, acc) -> int:
    """E of a valid ``choice_score`` call; ValueError otherwise."""
    _tensor(loss, "loss", torch.float32, 1)
    _tensor(spans, "spans", torch.int32, 3, 8)
    E = spans.shape[0]
    _need(E >= 1, "choice_score needs E >= 1 examples")
    _need(tuple(spans.shape) == (E, CHOICES, 2), f"spans must be [E, {CHOICES}, 2], not {tuple(spans.shape)}")
    _tensor(labels, "labels", torch.int32, 1)
    _need(labels.numel() == E, f"labels must hold {E} elements, not {labels.numel()}")
    _tensor(mean, "mean", torch.float32, 2)
    _need(tuple(mean.shape) == (E, CHOICES), f"mean must be [{E}, {CHOICES}], not {tuple(mean.shape)}")
    _tensor(acc, "acc", torch.float64, 1)
    _need(acc.numel() == 2, f"acc must hold 2 elements, not {acc.numel()}")
    return E


def choice_score(loss, spans, labels, mean, acc):
    """mean[e, c] <- the mean of loss[first, first + n) over the span (first, n) = spans[e, c] of each completion (the
    per-token NLL ``xent_finish`` leaves; every span must lie inside ``loss`` with n >= 1); acc (fp64 [2]) += (examples
    whose lowest mean -- the first on a tie -- is at labels[e], examples)."""
    E = check_choice_score(loss, spans, labels, mean, acc)
    lib.call("aitj_choice_score", loss.data_ptr(), spans.data_ptr(), labels.data_ptr(), E, mean.data_ptr(),
             acc.data_ptr(), _stream())
    return mean
