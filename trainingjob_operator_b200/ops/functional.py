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
        assert colsum.dtype == torch.float32 and colsum.numel() == N and out.dtype == torch.bfloat16
        lib.load().aitj_gemm_set_colsum(colsum.data_ptr())
    lib.call("aitj_gemm_bf16", a.data_ptr(), b.data_ptr(), out.data_ptr(), M, N, K, a.stride(0), b.stride(0),
             out.stride(0), int(a_mn), int(b_mn), _ptr(bias), _ptr(residual), _ptr(aux), flags, int(split_k),
             int(block_n), int(max_ctas), _stream())
    return out


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
