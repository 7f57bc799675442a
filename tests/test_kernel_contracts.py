"""The CPU suite's kernel stand-ins (``tests/kernel_emulation.py``) refuse what the kernel library refuses.

Most tests run the engines with the entry points of ``ops/functional.py`` replaced by plain-PyTorch stand-ins.  A call
the library answers with an error code must fail there too, or an engine change passes on the CPU and fails on the
H100.  ``kernel_emulation.REFUSALS`` mirrors every host-side refusal of the library, keyed by (function, code):
- the parity test makes one bad call per row and requires the library's code from both the real entry point and the
  stand-in;
- the coverage test parses the ``extern "C"`` functions of ``ops/csrc/*.cu`` and requires a row for every ``return -N``
  that refuses arguments.

The library checks its arguments before it touches the device, so the real half runs on any machine: on a CPU box
with host tensors and a null stream, on a GPU box with device tensors.  Every buffer is padded so that the call would
stay in bounds if the library stopped refusing it; a change in the library then fails an assertion, never faults.
"""
import ctypes
import os
import re

import pytest
import torch

import kernel_emulation as ke
from trainingjob_operator_b200.ops import functional as F

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "trainingjob_operator_b200", "ops",
                    "csrc")
DEV = "cuda" if torch.cuda.is_available() else "cpu"

# Codes that report a failed CUDA runtime or driver call, not a refused argument: the tensor-map encoder missing from
# the driver (-10), cudaFuncSetAttribute (-20), a failed launch (-30), and the peer tables' cudaMemcpyToSymbol (-2 of
# the set_peers functions).  The encoder's own failures are returned as offsets from the driver's CUresult, never as a
# literal; the library refuses what the encoder would reject (misaligned TMA operands) by an explicit check first.
NOT_REFUSALS = {-10, -20, -30}
CUDA_FAILURES = {("aitj_gemm_set_peers", -2), ("aitj_fused_set_peers", -2)}

# Rows whose library half is skipped on a GPU: if the library stopped refusing these calls, the kernel would fault
# (a multimem store to an ordinary address, an add through an unset peer table).
FAULTS_IF_ACCEPTED = {("aitj_mc_push", -1), ("aitj_peer_push", -1)}


def _buf(shape, dtype=torch.bfloat16, offset=0):
    """A tensor of ``shape`` ``offset`` elements into a zeroed allocation with 4 KB to spare at the end."""
    n = 1
    for s in shape:
        n *= s
    pad = 4096 // torch.empty((), dtype=dtype).element_size()
    return torch.zeros(n + offset + pad, dtype=dtype, device=DEV)[offset:offset + n].view(*shape)


def _gemm_raw(M=128, N=128, K=128, flags=0, a_mn=0, b_mn=0, split_k=1, block_n=0, colsum=None, xent=None):
    """A direct ``aitj_gemm_bf16`` call: (setup of the one-shot buffers, positional arguments, the same arguments
    named for the table, the one-shot buffers named for the table)."""
    a, b, out = _buf((M, K)), _buf((N, K)), _buf((M, N), torch.float32)
    named = dict(A=a.data_ptr(), B=b.data_ptr(), out=out.data_ptr(), M=M, N=N, K=K, lda=K, ldb=K, ldc=N, a_mn=a_mn,
                 b_mn=b_mn, bias=0, residual=0, aux=0, flags=flags, split_k=split_k, block_n=block_n, max_ctas=0)
    extra = dict(colsum=0, xent_target=0, xent_part=0, xent_tgt=0, vocab=0)
    keep = [a, b, out]

    def setup(L):
        if colsum:
            cs = _buf((N,), torch.float32)
            keep.append(cs)
            extra["colsum"] = cs.data_ptr()
            L.aitj_gemm_set_colsum(ctypes.c_void_p(cs.data_ptr()))
        if xent:
            t, part, tl = _buf((M,), torch.int64), _buf((M, F.xent_blocks(N), 2), torch.float32), _buf((M,), torch.float32)
            keep.extend((t, part, tl))
            extra.update(xent_target=t.data_ptr(), xent_part=part.data_ptr(), xent_tgt=tl.data_ptr(), vocab=xent)
            L.aitj_gemm_set_xent(ctypes.c_void_p(t.data_ptr()), ctypes.c_void_p(part.data_ptr()),
                                 ctypes.c_void_p(tl.data_ptr()), xent)

    return setup, list(named.values()), named, extra


def _attn(T=128, B=1, H=1, causal=True, qkv_off=0, ds_off=None, bwd=False):
    """Functional arguments of attention_fwd / attention_bwd; buffers are sized for max(T, 128)."""
    rows = B * max(T, 128)
    qkv = _buf((rows, 3 * H * 64), offset=qkv_off)[:B * T]
    out = _buf((rows, H * 64))[:B * T]
    lse = _buf((B * H * max(T, 128),), torch.float32)[:B * H * T]
    ds = None if ds_off is None else _buf((rows,), torch.int32, offset=ds_off)[:B * T]
    if not bwd:
        return (qkv, out, lse, B, T, H), dict(causal=causal, doc_start=ds)
    d_out, delta = _buf((rows, H * 64))[:B * T], _buf((B * H * max(T, 128),), torch.float32)[:B * H * T]
    dq_acc, d_qkv = _buf((rows, H * 64), torch.float32)[:B * T], _buf((rows, 3 * H * 64))[:B * T]
    return (qkv, out, d_out, lse, delta, dq_acc, d_qkv, B, T, H), dict(causal=causal, doc_start=ds)


def _adamw(n):
    kw = dict(lr=1e-3)
    return (_buf((n,), torch.float32), _buf((n,), torch.float32), _buf((n,), torch.float32),
            _buf((n,), torch.float32), _buf((n,)), _buf(((n + 255) // 256,), torch.uint8)), kw


def _peers(n):
    delta, bound = (ctypes.c_longlong * 8)(), (ctypes.c_longlong * 9)()
    return [None, delta, bound, n], dict(n=n)


# One bad call per row.  A functional case is (entry point, args, kwargs), made by both ``F`` and the stand-in.  Where
# functional.py refuses the arguments itself before the library sees them, the case is ("raw", ...): the library
# function is called directly, the stand-in's table consulted with the same arguments, and the functional entry point
# and its stand-in must raise alike for ``pre`` (the wrapper's own check), when one is given.
def _cases():
    def tok():
        return _buf((8,), torch.int64)

    return {
        ("aitj_gemm_bf16", -8): lambda: ("raw", "aitj_gemm_bf16", *_gemm_raw(flags=F.EPI_XENT | F.EPI_BIAS, xent=128),
                                         None),
        ("aitj_gemm_bf16", -1): lambda: ("gemm", (_buf((128, 128)), _buf((12, 128)), _buf((128, 12))), {}),
        ("aitj_gemm_bf16", -4): lambda: ("gemm", (_buf((128, 128)), _buf((128, 128)), _buf((128, 128), offset=1)), {}),
        ("aitj_gemm_bf16", -2): lambda: ("gemm", (_buf((128, 128)), _buf((128, 128)), _buf((128, 128), torch.float32)),
                                         dict(split_k=2)),
        ("aitj_gemm_bf16", -5): lambda: ("raw", "aitj_gemm_bf16",
                                         *_gemm_raw(flags=F.EPI_OUT_F32 | F.EPI_PEER, a_mn=1, b_mn=1), None),
        ("aitj_gemm_bf16", -3): lambda: ("gemm", (_buf((128, 128)), _buf((128, 128)), _buf((128, 128))),
                                         dict(block_n=64)),
        ("aitj_gemm_bf16", -6): lambda: ("raw", "aitj_gemm_bf16", *_gemm_raw(flags=F.EPI_OUT_F32, colsum=True), None),
        ("aitj_gemm_bf16", -7): lambda: ("gemm", (_buf((256, 128)), _buf((256, 128)), _buf((128, 128))),
                                         dict(a_mn=True, b_mn=True, bias=_buf((128,)))),
        ("aitj_gemm_set_peers", -1): lambda: ("raw", "aitj_gemm_set_peers", None, *_peers(0), {},
                                              ("FakeWorld", (0,), {})),
        ("aitj_fused_set_peers", -1): lambda: ("raw", "aitj_fused_set_peers", None, *_peers(0), {},
                                               ("FakeWorld", (0,), {})),
        ("aitj_attn_fwd", -1): lambda: ("attention_fwd", *_attn(T=64)),
        ("aitj_attn_fwd", -5): lambda: _attn_raw("aitj_attn_fwd", causal=False, ds_off=0),
        ("aitj_attn_fwd", -4): lambda: ("attention_fwd", *_attn(qkv_off=1)),
        ("aitj_attn_bwd", -1): lambda: ("attention_bwd", *_attn(T=64, bwd=True)),
        ("aitj_attn_bwd", -5): lambda: _attn_raw("aitj_attn_bwd", causal=False, ds_off=0),
        ("aitj_attn_bwd", -4): lambda: ("attention_bwd", *_attn(qkv_off=1, bwd=True)),
        ("aitj_layernorm_fwd", -1): lambda: ("layernorm_fwd", (_buf((8, 1280)), _buf((1280,)), _buf((1280,)),
                                                               _buf((8, 1280)), _buf((8,), torch.float32),
                                                               _buf((8,), torch.float32)), {}),
        ("aitj_layernorm_bwd", -1): lambda: ("layernorm_bwd", (_buf((8, 1536)), _buf((8, 1536)), _buf((1536,)),
                                                               _buf((8,), torch.float32), _buf((8,), torch.float32),
                                                               _buf((8, 1536)), _buf((1536,), torch.float32),
                                                               _buf((1536,), torch.float32)), {}),
        ("aitj_embedding_fwd", -1): lambda: ("embedding_fwd", (tok(), _buf((16, 12)), _buf((8, 12)), _buf((8, 12)), 8), {}),
        ("aitj_embedding_bwd", -1): lambda: ("embedding_bwd", (tok(), _buf((8, 6)), _buf((16, 6), torch.float32),
                                                               _buf((8, 6), torch.float32), 8), {}),
        ("aitj_embedding3_fwd", -1): lambda: ("embedding3_fwd", (tok(), tok(), _buf((16, 12)), _buf((8, 12)), _buf((2, 12)),
                                                                 _buf((8, 12)), 8), {}),
        ("aitj_embedding3_bwd", -1): lambda: ("embedding3_bwd", (tok(), tok(), _buf((8, 6)), _buf((16, 6), torch.float32),
                                                                 _buf((8, 6), torch.float32),
                                                                 _buf((2, 6), torch.float32), 8), {}),
        ("aitj_softmax_xent", -1): lambda: ("softmax_xent", (_buf((2, 12)), tok()[:2], _buf((2,), torch.float32), 10, 1.0),
                                            {}),
        ("aitj_softmax_xent", -2): lambda: ("softmax_xent", (_buf((1, 102408)), tok()[:1], _buf((1,), torch.float32),
                                                             102408, 1.0), {}),
        ("aitj_xent_finish", -1): lambda: ("xent_finish", (_buf((4, 0, 2), torch.float32), _buf((4,), torch.float32),
                                                           tok()[:4], _buf((4,), torch.float32),
                                                           _buf((2,), torch.float64)), {}),
        ("aitj_colsum", -1): lambda: ("colsum", (_buf((8, 12)), _buf((12,), torch.float32)), {}),
        ("aitj_qkv_gather_colsum", -1): lambda: ("qkv_gather_colsum", (_buf((1, 2, 8, 4)), _buf((1, 2, 8, 4)),
                                                                       _buf((1, 2, 8, 4)), _buf((8, 24)),
                                                                       _buf((24,), torch.float32)), {}),
        ("aitj_sumsq", -1): lambda: ("sumsq", (_buf((6,), torch.float32), _buf((1,), torch.float32)), {}),
        ("aitj_peer_push", -1): lambda: ("peer_push", (_buf((6,), torch.float32), _buf((6,), torch.float32)), {}),
        ("aitj_adamw", -1): lambda: ("adamw", *_adamw(260)),
        ("aitj_mc_push", -1): lambda: ("mc_push", (_buf((8,), torch.float32).data_ptr(), _buf((8,), torch.float32), 6),
                                       {}),
        ("aitj_cast_f32_bf16", -1): lambda: ("cast_f32_bf16", (_buf((6,), torch.float32), _buf((6,))), {}),
        ("aitj_gelu_fwd", -1): lambda: ("gelu_fwd", (_buf((12,)), _buf((12,))), {}),
        ("aitj_gelu_bwd", -1): lambda: ("gelu_bwd", (_buf((12,)), _buf((12,)), _buf((12,))), {}),
    }


def _attn_raw(fn, causal, ds_off):
    """A direct attention call with a document mask: functional.py refuses these itself (ValueError)."""
    bwd = fn == "aitj_attn_bwd"
    args, kw = _attn(bwd=bwd, causal=causal, ds_off=ds_off)
    ds = kw["doc_start"]
    ptrs = [t.data_ptr() for t in args[:-3]]
    B, T, H = args[-3:]
    pos = ptrs + [ds.data_ptr(), B, T, H, int(causal), 0.0]
    named = dict(qkv=ptrs[0], out=ptrs[1], d_out=ptrs[2] if bwd else 0, doc_start=ds.data_ptr(), B=B, T=T, H=H,
                 causal=int(causal))
    return ("raw", fn, None, pos, named, {}, ("attention_bwd" if bwd else "attention_fwd", args, kw))


@pytest.fixture
def lib(monkeypatch):
    if DEV == "cpu":
        monkeypatch.setattr(F, "_stream", lambda: 0)    # the refusals come before any CUDA call
    return F.lib.load(build_if_missing=False)


def _code(e):
    return e.code if isinstance(e, F.lib.KernelError) else repr(e)


def _raises(fn, *a, **kw):
    try:
        fn(*a, **kw)
    except Exception as e:  # noqa: BLE001
        return e
    return None


def _real_and_emulated(key, L, real_half=True):
    """(exception of the library side, exception of the stand-in side) for the case of table row ``key``."""
    case = _cases()[key]()
    if case[0] != "raw":
        entry, args, kw = case
        return (_raises(getattr(F, entry), *args, **kw) if real_half else None), _raises(getattr(ke, entry), *args, **kw)
    _, fn, setup, pos, named, extra, pre = case
    real = None
    if real_half:
        if setup is not None:
            setup(L)
        stream = None if DEV == "cpu" else torch.cuda.current_stream().cuda_stream
        real = _raises(F.lib.call, fn, *(list(pos) if fn.endswith("set_peers") else list(pos) + [stream]))
    if pre is not None and pre[0] == "FakeWorld":     # the stand-in of ShardedGradState installs both peer tables
        assert _code(_raises(ke.FakeWorld, *pre[1])) == key[1]
    elif pre is not None:                             # the wrapper refuses first; the stand-in must too, alike
        entry, args, kw = pre
        a, b = _raises(getattr(F, entry), *args, **kw), _raises(getattr(ke, entry), *args, **kw)
        assert type(a) is type(b) and a is not None and str(a) == str(b), (a, b)
    return real, _raises(ke.refuse, fn, **named, **extra)


@pytest.mark.parametrize("key", sorted(_cases()), ids=lambda k: f"{k[0]}{k[1]}")
def test_the_stand_in_refuses_what_the_library_refuses(lib, key):
    # on a GPU, the library half of a call that would fault if accepted is left out; the stand-in half still runs
    real_half = not (DEV == "cuda" and key in FAULTS_IF_ACCEPTED)
    real, emulated = _real_and_emulated(key, lib, real_half)
    assert _code(emulated) == key[1], f"the stand-in's answer to the bad call of {key}: {emulated!r}"
    if real_half:
        assert _code(real) == key[1], f"the library's answer to the bad call of {key}: {real!r}"


def test_every_row_has_a_bad_call():
    assert set(_cases()) == set(ke.REFUSALS)
    assert all(reason and callable(bad) for reason, bad in ke.REFUSALS.values())


def library_refusals():
    """{(function, code)} of every literal ``return -N`` inside the ``extern "C"`` functions of ops/csrc/*.cu."""
    out = set()
    for name in sorted(os.listdir(CSRC)):
        if not name.endswith(".cu"):
            continue
        src = open(os.path.join(CSRC, name)).read()
        for block in re.findall(r'extern "C" \{(.*?)\}\s*// extern "C"', src, re.S):
            parts = re.split(r"^int (aitj_\w+)\(", block, flags=re.M)
            for fn, body in zip(parts[1::2], parts[2::2]):
                # `return -N;` and the failure arm of a conditional, `... ? 0 : -N;`
                out |= {(fn, -int(n)) for n in re.findall(r"(?:return|\? 0 :)\s*-(\d+)\s*;", body)}
    return out


def test_every_library_refusal_has_a_row():
    found = library_refusals()
    assert len({fn for fn, _ in found}) >= 20, "the parser lost the library's entry points"
    missing = sorted(k for k in found if k[1] not in NOT_REFUSALS and k not in CUDA_FAILURES and k not in ke.REFUSALS)
    assert not missing, f"refusals of the library without a row in kernel_emulation.REFUSALS: {missing}"
    assert CUDA_FAILURES <= found
    stale = sorted(set(ke.REFUSALS) - found)
    assert not stale, f"rows of kernel_emulation.REFUSALS the library no longer has: {stale}"


def test_a_refused_gemm_does_not_hand_its_column_sums_to_the_next(lib):
    """The column-sum buffer is one-shot: a GEMM refused before reaching it must still consume it.  Here the second
    call (an fp32 output, which takes no column sums) would otherwise be refused for column sums (-6) it never asked
    for; without them it is refused for the kernel it lacks (-7), both before the device is touched."""
    cs = _buf((128,), torch.float32)
    with pytest.raises(F.lib.KernelError) as e:
        F.gemm(_buf((128, 128)), _buf((128, 128)), _buf((128, 128), offset=1), colsum=cs)
    assert e.value.code == F.GEMM_MISALIGNED
    with pytest.raises(F.lib.KernelError) as e:
        F.gemm(_buf((128, 128)), _buf((128, 128)), _buf((128, 128), torch.float32), a_mn=True, b_mn=True,
               bias=_buf((128,)))
    assert e.value.code == F.GEMM_NO_KERNEL


def test_the_gemm_stand_in_takes_column_sums_at_every_tile():
    """The kernel forms column sums in all four tile configurations, so the stand-in accepts each."""
    a, w = torch.randn(128, 256).bfloat16(), torch.randn(256, 256).bfloat16()
    for bn in (0, 128, 256, 512, 1024):
        out, cs = torch.empty(128, 256, dtype=torch.bfloat16), torch.ones(256)
        ke.gemm(a, w, out, b_mn=True, dgelu=True, aux=torch.randn(128, 256).bfloat16(), colsum=cs, block_n=bn)
        torch.testing.assert_close(cs, 1 + out.float().sum(0))


@pytest.mark.gpu
def test_a_refused_adamw_sweep_does_not_hand_its_shard_settings_to_the_next():
    """``adamw(sumsq_n=...)`` sets the number of partial square sums for the next sweep only.  A sweep the library
    refuses must consume it too: here a leaked count of 2 would add the second partial (1e6) to the norm and clip."""
    n = 256

    def sweep(after_refusal):
        torch.manual_seed(0)
        p, g = torch.randn(n, device="cuda"), torch.randn(n, device="cuda")
        m, v, p16 = torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda"), torch.empty(n, device="cuda").bfloat16()
        wd = torch.ones(1, dtype=torch.uint8, device="cuda")
        sq = torch.tensor([1.0, 1e6], device="cuda")
        if after_refusal:
            bad = _adamw(n + 4)[0]
            with pytest.raises(F.lib.KernelError) as e:
                F.adamw(*bad, lr=1e-3, sumsq_n=2)
            assert e.value.code == -1
        F.adamw(p, g, m, v, p16, wd, lr=1e-2, step=1, sumsq_buf=sq, max_norm=2.0)
        torch.cuda.synchronize()
        return p

    assert torch.equal(sweep(False), sweep(True))


# ------------------------------------------------------------------------------------ side effects, on the device
# The kernel and its stand-in run on deep copies of the same device inputs.  Outputs the call overwrites start as NaN,
# outputs it adds into start as 1000 + noise (an overwrite then misses by ~1000).  Afterwards every tensor argument is
# compared: inputs must be untouched on both sides, accumulators within a summation-order bound n * 2^-23 * sum|terms|
# (the starting value counted as a term), bf16 outputs within 2 bf16 ulps of max(|stand-in|, rms).
EPS32 = 2.0 ** -23


def _acc(n):
    return 1000.0 + torch.randn(n, device="cuda")


def _bf16_ulps(got, want):
    """|got - want| in bf16 ulps of max(|want|, rms(want)), elementwise."""
    w = want.float()
    scale = torch.maximum(w.abs(), w.pow(2).mean().sqrt())
    ulp = torch.exp2(torch.floor(torch.log2(scale.clamp_min(1e-30))) - 7)
    return (got.float() - w).abs() / ulp


def _within(name, got, want, bound):
    d = (got.double() - want.double()).abs()
    worst = float((d / bound.double().clamp_min(1e-300)).max())
    assert bool(torch.isfinite(got).all()) and worst <= 1.0, f"{name}: worst |kernel - stand-in| / bound = {worst:.3g}"
    return worst


def _run_both(entry, args):
    real, emu = copy_args(args), copy_args(args)
    getattr(F, entry)(**real)
    getattr(ke, entry)(**emu)
    torch.cuda.synchronize()
    return real, emu


def copy_args(args):
    import copy

    return copy.deepcopy(args)


def _untouched(args, real, emu, names):
    for n in names:
        assert torch.equal(real[n], args[n]) and torch.equal(emu[n], args[n]), f"input {n} was written"


def _case_colsum():
    M, N = 257, 264
    args = dict(dy=torch.randn(M, N, device="cuda").bfloat16(), db=_acc(N))
    real, emu = _run_both("colsum", args)
    _untouched(args, real, emu, ["dy"])
    terms = args["dy"].double().abs().sum(0) + args["db"].double().abs()
    return {"db": _within("colsum db", real["db"], emu["db"], (M + 1) * EPS32 * terms)}


def _case_layernorm_bwd():
    M, C = 64, 256
    x = torch.randn(M, C, device="cuda").bfloat16()
    xf = x.float()
    mean, rstd = xf.mean(1), torch.rsqrt(xf.var(1, unbiased=False) + 1e-5)
    args = dict(dy=torch.randn(M, C, device="cuda").bfloat16(), x=x,
                gamma=(1 + 0.1 * torch.randn(C, device="cuda")).bfloat16(), mean=mean, rstd=rstd,
                dx=torch.full((M, C), float("nan"), device="cuda").bfloat16(), dgamma=_acc(C), dbeta=_acc(C),
                dres=None, dxsum=_acc(C))
    real, emu = _run_both("layernorm_bwd", args)
    _untouched(args, real, emu, ["dy", "x", "gamma", "mean", "rstd"])
    out = {"dx": float(_bf16_ulps(real["dx"], emu["dx"]).max()) / 2}
    assert out["dx"] <= 1.0, f"layernorm_bwd dx: {2 * out['dx']:.3g} bf16 ulps"
    h = ((xf - mean[:, None]) * rstd[:, None]).double()
    d = args["dy"].double()
    out["dgamma"] = _within("dgamma", real["dgamma"], emu["dgamma"],
                            (M + 1) * EPS32 * ((d * h).abs().sum(0) + args["dgamma"].double().abs()))
    out["dbeta"] = _within("dbeta", real["dbeta"], emu["dbeta"],
                           (M + 1) * EPS32 * (d.abs().sum(0) + args["dbeta"].double().abs()))
    # dxsum sums dx before or after its bf16 rounding: the two sides may differ by their dx's and by one rounding each
    dx_diff = (real["dx"].double() - emu["dx"].double()).abs().sum(0)
    rounding = 2.0 ** -8 * emu["dx"].double().abs().sum(0)
    out["dxsum"] = _within("dxsum", real["dxsum"], emu["dxsum"],
                           (M + 1) * EPS32 * (emu["dx"].double().abs().sum(0) + args["dxsum"].double().abs())
                           + dx_diff + rounding)
    return out


def _case_gemm_xent():
    M, K, N, V = 300, 64, 520, 389
    target = torch.randint(0, V, (M,), device="cuda")
    target[::9] = -1
    args = dict(x=torch.randn(M, K, device="cuda").bfloat16(), w=(torch.randn(N, K, device="cuda") * 0.5).bfloat16(),
                target=target, vocab=V, part=torch.full((M, F.xent_blocks(N), 2), float("nan"), device="cuda"),
                tgt_logit=torch.full((M,), float("nan"), device="cuda"), block_n=512)
    real, emu = _run_both("gemm_xent", args)
    _untouched(args, real, emu, ["x", "w", "target"])
    dead = target < 0
    for side in (real, emu):       # rows without a target keep their sentinel
        assert bool(side["part"][dead].isnan().all()) and bool(side["tgt_logit"][dead].isnan().all()), \
            "rows without a target must keep their sentinel"
    live = ~dead
    zb = K * EPS32 * (args["x"].double().abs() @ args["w"].double().abs().t())       # per logit
    zb_row = zb.max(1).values[live]
    t = target[live]
    out = {"tgt_logit": _within("tgt_logit", real["tgt_logit"][live], emu["tgt_logit"][live],
                                zb[live].gather(1, t[:, None])[:, 0])}
    mx_real, mx_emu = real["part"][live][..., 0], emu["part"][live][..., 0]
    empty = torch.isinf(mx_emu)                        # blocks without a vocabulary column: -inf on both sides
    assert torch.equal(mx_real[empty], mx_emu[empty])
    out["max"] = _within("part max", mx_real[~empty], mx_emu[~empty],
                         zb_row[:, None].expand(-1, F.xent_blocks(N))[~empty])
    # sum of exp(z - max) over 128 columns: each exponent off by up to 2 zb, each exp2 approximation by 2 ulps
    s = emu["part"][live][..., 1].double()
    out["sumexp"] = _within("part sumexp", real["part"][live][..., 1], emu["part"][live][..., 1],
                            s * (4 * zb_row[:, None] + 128 * 2 * EPS32))
    return out


def _case_adamw():
    n = 1024
    g = torch.randn(n, device="cuda")
    args = dict(p=torch.randn(n, device="cuda"), g=g, m=0.1 * torch.randn(n, device="cuda"),
                v=0.01 * torch.rand(n, device="cuda"), p16=torch.full((n,), float("nan"), device="cuda").bfloat16(),
                wd_mask=torch.tensor([1, 0, 1, 0], dtype=torch.uint8, device="cuda"), lr=1e-2, step=3,
                sumsq_buf=(g * g).sum().reshape(1), max_norm=1.0, zero_grad=True)
    real, emu = _run_both("adamw", args)
    _untouched(args, real, emu, ["wd_mask", "sumsq_buf"])
    for side in (real, emu):
        assert bool((side["g"] == 0).all()), "the sweep must leave g zero"
        assert torch.equal(side["p16"], side["p"].bfloat16()), "p16 must be bf16(p)"
    # about 16 fp32 operations per element (clip, moments, bias corrections, sqrt, division, decay)
    p0, m0, v0 = args["p"].double().abs(), args["m"].double().abs(), args["v"].double().abs()
    return {"p": _within("adamw p", real["p"], emu["p"], 16 * EPS32 * (p0 + (emu["p"].double() - args["p"].double()).abs())),
            "m": _within("adamw m", real["m"], emu["m"], 16 * EPS32 * (m0 + g.double().abs())),
            "v": _within("adamw v", real["v"], emu["v"], 16 * EPS32 * (v0 + g.double() ** 2))}


def _case_attention_bwd():
    from trainingjob_operator_b200.ops.selfcheck import _check

    B, T, H = 1, 256, 2
    qkv = torch.randn(B * T, 3 * H * 64, device="cuda").bfloat16()
    out = torch.empty(B * T, H * 64, device="cuda").bfloat16()
    lse = torch.empty(B, H, T, device="cuda")
    F.attention_fwd(qkv, out, lse, B, T, H, causal=True)
    args = dict(qkv=qkv, out=out, d_out=torch.randn(B * T, H * 64, device="cuda").bfloat16(), lse=lse,
                delta=torch.zeros(B, H, T, device="cuda"), dq_acc=torch.zeros(B * T, H * 64, device="cuda"),
                d_qkv=torch.full((B * T, 3 * H * 64), float("nan"), device="cuda").bfloat16(), B=B, T=T, H=H)
    real, emu = _run_both("attention_bwd", args)       # delta is the kernel's scratch: not compared
    _untouched(args, real, emu, ["qkv", "out", "d_out", "lse"])
    for side in (real, emu):
        assert bool((side["dq_acc"] == 0).all()), "dq_acc must be zero again on exit"
    # the selfcheck's bound for the attention backward against an fp32 reference
    assert _check("attention_bwd d_qkv kernel vs stand-in", real["d_qkv"], emu["d_qkv"], 2e-2, rtol=5e-2,
                  atol_scale=1.5e-1)
    return {}


def _case_gemm_colsum():
    out = {}
    M, N, K = 256, 512, 192
    for bn in (0, 128, 256, 512, 1024):
        args = dict(a=torch.randn(M, K, device="cuda").bfloat16(), b=(torch.randn(K, N, device="cuda") * 0.1).bfloat16(),
                    out=torch.full((M, N), float("nan"), device="cuda").bfloat16(), b_mn=True, dgelu=True,
                    aux=torch.randn(M, N, device="cuda").bfloat16(), colsum=_acc(N), block_n=bn)
        real, emu = _run_both("gemm", args)
        _untouched(args, real, emu, ["a", "b", "aux"])
        # the colsum is the column sum of the stored output (summed before or after its rounding), on each side
        for tag, side in (("kernel", real), ("stand-in", emu)):
            o = side["out"].double()
            bound = (M + 1) * EPS32 * (o.abs().sum(0) + args["colsum"].double().abs()) + 2.0 ** -9 * o.abs().sum(0)
            out[f"colsum {tag} bn={bn}"] = _within(f"colsum {tag} bn={bn}", side["colsum"] - args["colsum"],
                                                   o.sum(0), bound)
    return out


SIDE_EFFECT_CASES = {"colsum": _case_colsum, "layernorm_bwd": _case_layernorm_bwd, "gemm_xent": _case_gemm_xent,
                     "adamw": _case_adamw, "attention_bwd": _case_attention_bwd, "gemm_colsum": _case_gemm_colsum}


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(SIDE_EFFECT_CASES))
def test_the_stand_in_has_the_kernels_side_effects(case):
    worst = SIDE_EFFECT_CASES[case]()
    print(f"{case}: " + ", ".join(f"{k} {v:.3g}" for k, v in worst.items()))
