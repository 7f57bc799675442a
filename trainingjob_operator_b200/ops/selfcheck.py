"""Numerics self-check of every hand-written kernel against a plain fp32 PyTorch reference.

Run as ``python -m trainingjob_operator_b200.ops.selfcheck --case <name>`` (one process per
case: a trapping kernel poisons its CUDA context, so cases are isolated) or ``--case all``.
Exit code 0 = pass.  ``tests/test_gpu_kernels.py`` drives it under ``@pytest.mark.gpu``.
"""
from __future__ import annotations

import argparse
import os
import sys
import time

import torch

# The engine cases compare against tolerances that were settled on the weights a CPU generator draws for these seeds;
# workers initialise on the device (models/flat_params.py), the self-check keeps the draw it was validated with.
os.environ.setdefault("AITJ_PARAM_INIT", "cpu")

from . import functional as F


def _rel_err(got: torch.Tensor, ref: torch.Tensor) -> float:
    got = got.float()
    ref = ref.float()
    return float((got - ref).norm() / (ref.norm() + 1e-12))


def _rand(*shape, scale=1.0, dtype=torch.bfloat16):
    return (torch.randn(*shape, device="cuda", dtype=torch.float32) * scale).to(dtype)


def _check(name, got, ref, tol, rtol=None, atol_scale=None):
    """Two oracles: the relative Frobenius error (catches a systematically wrong kernel) AND an element-wise bound
    |got - ref| <= atol + rtol * |ref| with atol tied to the spread of the reference (catches a single wrong row /
    column tail or one bad 32x64 store that would vanish inside the norm).  bf16 outputs of an fp32 accumulation differ
    from the fp32 reference of the same bf16 inputs by the output rounding (2^-9 relative) plus summation-order noise."""
    g, r = got.float(), ref.float()
    err = _rel_err(g, r)
    rtol = 2e-2 if rtol is None else rtol
    scale = float(r.std()) if r.numel() > 1 else float(r.abs().max())
    atol = (2e-2 if atol_scale is None else atol_scale) * max(scale, 1e-30)
    bad = (g - r).abs() > atol + rtol * r.abs()
    nbad = int(bad.sum())
    worst = float(((g - r).abs() - rtol * r.abs()).max()) if r.numel() else 0.0
    ok = err < tol and nbad == 0 and bool(torch.isfinite(g).all())
    where = ""
    if nbad:
        idx = bad.nonzero()[0].tolist()
        where = f" first bad element at {idx} got={float(g[tuple(idx)]):.4g} ref={float(r[tuple(idx)]):.4g}"
    print(f"  {name:<44s} rel_err={err:.3e} tol={tol:.1e} elementwise: {nbad} of {r.numel()} outside "
          f"atol={atol:.2e}+{rtol:.0e}*|ref| (worst excess {worst:.2e}) {'ok' if ok else 'FAIL'}{where}", flush=True)
    return ok


# ----------------------------------------------------------------------------- GEMM cases
def _gemm_case(M, N, K, a_mn, b_mn, **kw):
    a = _rand(K, M) if a_mn else _rand(M, K)
    b = _rand(K, N) if b_mn else _rand(N, K)
    A = (a.t() if a_mn else a).float()
    B = (b.t() if b_mn else b).float()
    ref = A @ B.t()
    out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    F.gemm(a, b, out, a_mn=a_mn, b_mn=b_mn, **kw)
    torch.cuda.synchronize()
    return _check(f"gemm M={M} N={N} K={K} a_mn={int(a_mn)} b_mn={int(b_mn)} {kw}", out, ref, 1e-2)


def case_gemm_tn():
    ok = True
    for (M, N, K) in [(128, 256, 64), (128, 128, 64), (256, 256, 128), (512, 768, 768), (1000, 776, 200),
                      (4096, 2304, 768), (384, 50304, 768)]:
        ok &= _gemm_case(M, N, K, False, False)
    ok &= _gemm_case(512, 512, 512, False, False, block_n=128)
    ok &= _gemm_case(2048, 768, 3072, False, False, max_ctas=7)
    return ok


def case_gemm_nn():
    ok = True
    for (M, N, K) in [(128, 256, 64), (256, 256, 256), (512, 768, 2304), (1000, 776, 200), (2048, 768, 50304 // 8)]:
        ok &= _gemm_case(M, N, K, False, True)
    ok &= _gemm_case(512, 512, 512, False, True, block_n=128)
    return ok


def case_gemm_tt():
    ok = True
    for (M, N, K) in [(128, 256, 64), (256, 256, 256), (2304, 768, 4096), (776, 1000, 200)]:
        ok &= _gemm_case(M, N, K, True, True)
    ok &= _gemm_case(256, 512, 512, True, False)
    ok &= _gemm_case(512, 512, 512, True, True, block_n=128)
    return ok


def case_gemm_epilogue():
    ok = True
    M, N, K = 512, 768, 768
    a, b = _rand(M, K), _rand(N, K, scale=0.05)
    bias = _rand(N)
    res = _rand(M, N)
    pre_ref = a.float() @ b.float().t() + bias.float()
    # bias + gelu + save_pre
    out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    aux = torch.empty_like(out)
    F.gemm(a, b, out, bias=bias, gelu=True, save_pre=True, aux=aux)
    ok &= _check("bias+gelu", out, torch.nn.functional.gelu(pre_ref, approximate="tanh"), 1e-2)
    ok &= _check("save_pre", aux, pre_ref, 1e-2)
    # bias + residual
    F.gemm(a, b, out, bias=bias, residual=res)
    ok &= _check("bias+residual", out, pre_ref + res.float(), 1e-2)
    # dgelu
    h = _rand(M, N)
    hf = h.float().requires_grad_(True)
    g = torch.nn.functional.gelu(hf, approximate="tanh")
    dy = a.float() @ b.float().t()
    (gref,) = torch.autograd.grad(g, hf, dy)
    F.gemm(a, b, out, dgelu=True, aux=h)
    ok &= _check("dgelu", out, gref, 1.5e-2)
    # fp32 store + accumulate with split-K
    o32 = torch.zeros(M, N, device="cuda", dtype=torch.float32)
    F.gemm(a, b, o32)
    ok &= _check("out_f32", o32, dy, 1e-2)
    o32.fill_(1.0)
    F.gemm(a, b, o32, accumulate=True, split_k=4)
    ok &= _check("accumulate split_k=4", o32, dy + 1.0, 1e-2)
    # wgrad-shaped: dW[N_out,K_in] += dy^T x
    Mtok, Nout, Kin = 4096, 768, 768
    dyv, x = _rand(Mtok, Nout), _rand(Mtok, Kin)
    dw = torch.zeros(Nout, Kin, device="cuda", dtype=torch.float32)
    sk = F.auto_split_k(Nout, Kin, Mtok)
    F.gemm(dyv, x, dw, a_mn=True, b_mn=True, accumulate=True, split_k=sk)
    ok &= _check(f"wgrad split_k={sk}", dw, dyv.float().t() @ x.float(), 1e-2)
    # owner-sharded weight gradient (EPI_PEER) with a second rank emulated on this GPU: the peer table maps the upper
    # half of the flat buffer to another local allocation standing in for rank 1's copy.  Rows this rank owns are summed
    # in place; the others arrive in the owner's copy, and the local copy of them is zero again afterwards.
    import ctypes

    ref = dyv.float().t() @ x.float()
    half = Nout // 2
    for sk_peer in (1, 4):
        local = torch.zeros(Nout * Kin, device="cuda")
        owner1 = torch.zeros(Nout * Kin, device="cuda")
        delta = (ctypes.c_longlong * 8)(0, owner1.data_ptr() - local.data_ptr(), *([0] * 6))
        bound = (ctypes.c_longlong * 9)(0, half * Kin, *([Nout * Kin] * 7))
        assert F.lib.load().aitj_gemm_set_peers(ctypes.c_void_p(local.data_ptr()), delta, bound, 2) == 0
        F.gemm(dyv, x, F.PeerView(local.view(Nout, Kin)), a_mn=True, b_mn=True, accumulate=True, split_k=sk_peer)
        torch.cuda.synchronize()
        lo, hi = local.view(Nout, Kin), owner1.view(Nout, Kin)
        ok &= _check(f"peer wgrad split_k={sk_peer}: owned rows in place", lo[:half], ref[:half], 1e-2)
        ok &= _check(f"peer wgrad split_k={sk_peer}: other rows at the owner", hi[half:], ref[half:], 1e-2)
        ok &= bool((lo[half:] == 0).all()) and bool((hi[:half] == 0).all())
    torch.cuda.synchronize()
    return ok


def case_gemm_quad():
    """4-CTA cluster kernel (two CTA pairs sharing the B tile by TMA multicast; block_n=1024): all layouts, odd numbers
    of 256-row tiles (one pair of the last cluster idles on an out-of-range tile), tails, split-K, fused epilogues."""
    ok = True
    for (M, N, K, a_mn, b_mn) in [(512, 256, 64, False, False), (512, 256, 768, False, False),
                                  (768, 512, 256, False, False), (1000, 776, 200, False, False),
                                  (4096, 2304, 768, False, False), (2048, 768, 3072, False, True),
                                  (1280, 520, 328, False, True), (2304, 768, 4096, True, True),
                                  (776, 1000, 200, True, True), (1024, 512, 512, True, False)]:
        ok &= _gemm_case(M, N, K, a_mn, b_mn, block_n=1024)
    ok &= _gemm_case(4096, 768, 768, False, False, block_n=1024, max_ctas=8)
    M, N, K = 1024, 768, 768
    a, b = _rand(M, K), _rand(N, K, scale=0.05)
    bias, res = _rand(N), _rand(M, N)
    pre_ref = a.float() @ b.float().t() + bias.float()
    out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    aux = torch.empty_like(out)
    F.gemm(a, b, out, bias=bias, gelu=True, save_pre=True, aux=aux, block_n=1024)
    ok &= _check("quad bias+gelu", out, torch.nn.functional.gelu(pre_ref, approximate="tanh"), 1e-2)
    ok &= _check("quad save_pre", aux, pre_ref, 1e-2)
    F.gemm(a, b, out, bias=bias, residual=res, block_n=1024)
    ok &= _check("quad bias+residual", out, pre_ref + res.float(), 1e-2)
    Mtok, Nout, Kin = 4096, 2304, 768
    dyv, x = _rand(Mtok, Nout), _rand(Mtok, Kin)
    dw = torch.ones(Nout, Kin, device="cuda", dtype=torch.float32)
    F.gemm(dyv, x, dw, a_mn=True, b_mn=True, accumulate=True, split_k=4, block_n=1024)
    ok &= _check("quad wgrad split_k=4", dw, dyv.float().t() @ x.float() + 1.0, 1e-2)
    torch.cuda.synchronize()
    return ok


def case_gemm_2cta():
    """CTA-pair kernel (wgmma, 256x256 tile per 2-CTA cluster): all layouts + epilogues."""
    ok = True
    for (M, N, K, a_mn, b_mn) in [(256, 256, 64, False, False), (256, 256, 256, False, False),
                                  (512, 768, 768, False, False), (1000, 776, 200, False, False),
                                  (4096, 2304, 768, False, False), (384, 50304, 768, False, False),
                                  (512, 768, 2304, False, True), (2048, 768, 6288, False, True),
                                  (2304, 768, 4096, True, True), (776, 1000, 200, True, True),
                                  (256, 512, 512, True, False)]:
        ok &= _gemm_case(M, N, K, a_mn, b_mn, block_n=512)
    ok &= _gemm_case(2048, 768, 3072, False, False, block_n=512, max_ctas=6)
    M, N, K = 1024, 768, 768
    a, b = _rand(M, K), _rand(N, K, scale=0.05)
    bias, res = _rand(N), _rand(M, N)
    pre_ref = a.float() @ b.float().t() + bias.float()
    out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    aux = torch.empty_like(out)
    F.gemm(a, b, out, bias=bias, gelu=True, save_pre=True, aux=aux, block_n=512)
    ok &= _check("2cta bias+gelu", out, torch.nn.functional.gelu(pre_ref, approximate="tanh"), 1e-2)
    ok &= _check("2cta save_pre", aux, pre_ref, 1e-2)
    F.gemm(a, b, out, bias=bias, residual=res, block_n=512)
    ok &= _check("2cta bias+residual", out, pre_ref + res.float(), 1e-2)
    Mtok, Nout, Kin = 4096, 768, 3072
    dyv, x = _rand(Mtok, Nout), _rand(Mtok, Kin)
    dw = torch.ones(Nout, Kin, device="cuda", dtype=torch.float32)
    F.gemm(dyv, x, dw, a_mn=True, b_mn=True, accumulate=True, split_k=4, block_n=512)
    ok &= _check("2cta wgrad split_k=4 (TMA reduce-add)", dw, dyv.float().t() @ x.float() + 1.0, 1e-2)
    # dgrad + dGELU with the bias gradient (column sums of the stored bf16 output) fused into the epilogue; M tail
    Md, Nd, Kd = 1000, 3072, 768
    dyd, wd, pre = _rand(Md, Kd), _rand(Kd, Nd, scale=0.05), _rand(Md, Nd)
    outd = torch.empty(Md, Nd, device="cuda", dtype=torch.bfloat16)
    cs = torch.full((Nd,), 2.0, device="cuda")
    F.gemm(dyd, wd, outd, b_mn=True, dgelu=True, aux=pre, block_n=512, colsum=cs)
    pf = pre.float().requires_grad_(True)
    (gp,) = torch.autograd.grad(torch.nn.functional.gelu(pf, approximate="tanh").sum(), pf)
    ok &= _check("2cta dgrad*dgelu", outd, (dyd.float() @ wd.float()) * gp, 2e-2)
    ok &= _check("2cta fused colsum (bias grad)", cs, outd.float().sum(0) + 2.0, 1e-3)
    torch.cuda.synchronize()
    return ok


# ----------------------------------------------------------------------------- fused ops
def case_fused_ops():
    ok = True
    torch.manual_seed(0)
    M, C = 1000, 768
    x = _rand(M, C)
    gamma, beta = _rand(C) + 1.0, _rand(C, scale=0.1)
    y = torch.empty_like(x)
    mean = torch.empty(M, device="cuda")
    rstd = torch.empty(M, device="cuda")
    F.layernorm_fwd(x, gamma, beta, y, mean, rstd)
    xf = x.float().requires_grad_(True)
    gf, bf = gamma.float().requires_grad_(True), beta.float().requires_grad_(True)
    yref = torch.nn.functional.layer_norm(xf, (C,), gf, bf, 1e-5)
    ok &= _check("layernorm fwd", y, yref, 1e-2)
    dy = _rand(M, C)
    dres = _rand(M, C)
    dx = torch.empty_like(x)
    dgamma = torch.zeros(C, device="cuda")
    dbeta = torch.zeros(C, device="cuda")
    dxsum = torch.zeros(C, device="cuda")
    F.layernorm_bwd(dy, x, gamma, mean, rstd, dx, dgamma, dbeta, dres=dres, dxsum=dxsum)
    gx, gg, gb = torch.autograd.grad(yref, (xf, gf, bf), dy.float())
    ok &= _check("layernorm bwd dxsum (bias grad)", dxsum, (gx + dres.float()).sum(0), 1e-2)
    ok &= _check("layernorm bwd dx(+dres)", dx, gx + dres.float(), 1e-2)
    ok &= _check("layernorm bwd dgamma", dgamma, gg, 1e-2)
    ok &= _check("layernorm bwd dbeta", dbeta, gb, 1e-2)

    # embedding
    V, T, B = 1024, 64, 8
    wte, wpe = _rand(V, C), _rand(T, C)
    tok = torch.randint(0, V, (B * T,), device="cuda")
    out = torch.empty(B * T, C, device="cuda", dtype=torch.bfloat16)
    F.embedding_fwd(tok, wte, wpe, out, T)
    pos = torch.arange(B * T, device="cuda") % T
    ok &= _check("embedding fwd", out, wte.float()[tok] + wpe.float()[pos], 1e-2)
    dxe = _rand(B * T, C)
    dwte = torch.zeros(V, C, device="cuda")
    dwpe = torch.zeros(T, C, device="cuda")
    F.embedding_bwd(tok, dxe, dwte, dwpe, T)
    rwte = torch.zeros(V, C, device="cuda").index_add_(0, tok, dxe.float())
    rwpe = torch.zeros(T, C, device="cuda").index_add_(0, pos, dxe.float())
    ok &= _check("embedding bwd dwte", dwte, rwte, 1e-3)
    ok &= _check("embedding bwd dwpe", dwpe, rwpe, 1e-3)

    # softmax cross entropy (padded vocab)
    Mx, Vv, Vp = 256, 50257, 50304
    logits = _rand(Mx, Vp, scale=2.0)
    tgt = torch.randint(0, Vv, (Mx,), device="cuda")
    lf = logits[:, :Vv].float().requires_grad_(True)
    lref = torch.nn.functional.cross_entropy(lf, tgt, reduction="none")
    (gl,) = torch.autograd.grad(lref.sum() / Mx, lf)
    loss = torch.empty(Mx, device="cuda")
    work = logits.clone()
    F.softmax_xent(work, tgt, loss, Vv, 1.0 / Mx)
    ok &= _check("xent loss", loss, lref, 1e-2)
    ok &= _check("xent dlogits", work[:, :Vv], gl, 2e-2)
    ok &= bool((work[:, Vv:] == 0).all())

    # colsum
    dyc = _rand(3000, 2304)
    db = torch.zeros(2304, device="cuda")
    F.colsum(dyc, db)
    ok &= _check("colsum", db, dyc.float().sum(0), 1e-3)

    # attention-backward gather fused with the qkv bias gradient (both source layouts cuDNN may return)
    Bq, Hq, Tq, Dq = 3, 12, 100, 64
    for layout in ("bhtd", "bthd"):
        if layout == "bhtd":
            srcs = [_rand(Bq, Hq, Tq, Dq) for _ in range(3)]
        else:
            srcs = [_rand(Bq, Tq, Hq, Dq).transpose(1, 2) for _ in range(3)]
        outq = torch.empty(Bq * Tq, 3 * Hq * Dq, device="cuda", dtype=torch.bfloat16)
        dbq = torch.zeros(3 * Hq * Dq, device="cuda")
        F.qkv_gather_colsum(srcs[0], srcs[1], srcs[2], outq, dbq)
        refq = torch.stack([t.transpose(1, 2) for t in srcs], dim=2).reshape(Bq * Tq, 3 * Hq * Dq)
        ok &= bool((outq == refq).all())
        ok &= _check(f"qkv_gather_colsum {layout}", dbq, refq.float().sum(0), 1e-3)

    # adamw vs torch.optim.AdamW, two steps, with decay mask
    n = 256 * 40
    p0 = torch.randn(n, device="cuda")
    mask = torch.zeros(n // 256, dtype=torch.uint8, device="cuda")
    mask[:20] = 1
    p = p0.clone()
    m = torch.zeros(n, device="cuda")
    v = torch.zeros(n, device="cuda")
    p16 = torch.empty(n, device="cuda", dtype=torch.bfloat16)
    pa = torch.nn.Parameter(p0[: 256 * 20].clone())
    pb = torch.nn.Parameter(p0[256 * 20:].clone())
    opt = torch.optim.AdamW([{"params": [pa], "weight_decay": 0.1}, {"params": [pb], "weight_decay": 0.0}], lr=1e-2,
                            betas=(0.9, 0.95), eps=1e-8)
    for step in (1, 2):
        g = torch.randn(n, device="cuda")
        pa.grad = g[: 256 * 20].clone()
        pb.grad = g[256 * 20:].clone()
        opt.step()
        gg = g.clone()
        F.adamw(p, gg, m, v, p16, mask, lr=1e-2, beta1=0.9, beta2=0.95, eps=1e-8, weight_decay=0.1, step=step)
        ok &= bool((gg == 0).all())
    ref = torch.cat([pa.detach(), pb.detach()])
    ok &= _check("adamw p", p, ref, 1e-5)
    ok &= _check("adamw p16", p16, ref, 1e-2)

    # sumsq + clipping path
    g = torch.randn(n, device="cuda")
    ss = torch.zeros(1, device="cuda")
    F.sumsq(g, ss)
    ok &= _check("sumsq", ss, (g * g).sum().reshape(1), 1e-4)

    # gelu standalone
    xg = _rand(4096, 3072)
    yg = torch.empty_like(xg)
    F.gelu_fwd(xg, yg)
    ok &= _check("gelu fwd", yg, torch.nn.functional.gelu(xg.float(), approximate="tanh"), 1e-2)
    torch.cuda.synchronize()
    return ok


def case_gpt2_engine():
    """Hand-written engine (wgmma GEMMs + fused kernels) vs the plain fp32 PyTorch model: loss and grads."""
    from ..models.gpt2 import GPT2Config, GPT2Engine, GPT2Reference

    ok = True
    cfg = GPT2Config(vocab_size=1000, n_layer=2, n_head=4, n_embd=256, block_size=128, name="t")
    B, T = 4, 128
    import os

    for backend, attn, attn_bwd in (("wgmma", "cudnn", "cudnn"), ("cublas", "cudnn", "cudnn"),
                                    ("wgmma", "wgmma", "cudnn"), ("wgmma", "wgmma", "wgmma")):
        os.environ["AITJ_ATTN"] = attn
        os.environ["AITJ_ATTN_BWD"] = attn_bwd
        eng = GPT2Engine(cfg, B, T, "cuda", seed=3, gemm_backend=backend)
        os.environ.pop("AITJ_ATTN", None)
        os.environ.pop("AITJ_ATTN_BWD", None)
        assert eng.attn_impl == attn and eng.attn_bwd_impl == attn_bwd
        backend = backend if attn == "cudnn" else backend + "+attn" + ("+attn_bwd" if attn_bwd == "wgmma" else "")
        ref = GPT2Reference(cfg, eng.params).cuda()
        g = torch.Generator().manual_seed(5)
        tok = torch.randint(0, cfg.vocab_size, (B, T), generator=g).cuda()
        tgt = torch.roll(tok, -1, dims=1)
        eng.tok.copy_(tok.view(-1)); eng.tgt.copy_(tgt.view(-1))
        eng.params.g32.zero_()
        eng.forward(); eng.backward()
        torch.cuda.synchronize()
        rl = ref(tok, tgt)
        rl.backward()
        ok &= _check(f"[{backend}] loss", eng.loss, rl.detach().reshape(1), 5e-3)
        for name in ("wte", "wpe", "h0.qkv_w", "h0.qkv_b", "h0.proj_w", "h0.fc_w", "h0.fc_b", "h0.fc2_w", "h1.ln1_w",
                     "h1.ln2_b", "h1.fc2_w", "lnf_w", "lnf_b"):
            gref = ref.p(name).grad
            if name == "wte":
                gref = gref.clone()
            # a whole bf16 forward + backward separates the engine from the fp32 model by rounding noise per element:
            # the element-wise bound is correspondingly wide here (it still catches a missing tile or a wrong row)
            ok &= _check(f"[{backend}] grad {name}", eng.params.grad(name), gref, 4e-2, rtol=1e-1, atol_scale=2.5e-1)
        # three optimizer steps must reduce the loss on a fixed batch
        l0 = float(eng.loss.item())
        for step in range(1, 4):
            eng.optimizer_step(lr=1e-3, step=step)
            eng.forward(); eng.backward()
        l1 = float(eng.loss.item())
        print(f"  [{backend}] loss {l0:.4f} -> {l1:.4f}")
        ok &= l1 < l0
    return ok


def case_attention_bwd():
    """wgmma flash-attention backward vs. autograd through an fp32 PyTorch attention on the same bf16 inputs (causal
    and full), plus its device time next to the cuDNN SDPA backward PyTorch dispatches to."""
    ok = True
    for (B, T, H, causal) in [(1, 128, 1, True), (2, 256, 3, True), (2, 384, 2, False), (1, 1024, 4, True)]:
        C = H * 64
        qkv = _rand(B * T, 3 * C, scale=1.0)
        d_out = _rand(B * T, C, scale=1.0)
        out = torch.empty(B * T, C, device="cuda", dtype=torch.bfloat16)
        lse = torch.empty(B, H, T, device="cuda")
        F.attention_fwd(qkv, out, lse, B, T, H, causal=causal)
        delta = torch.empty(B, H, T, device="cuda")
        dq_acc = torch.zeros(B * T, C, device="cuda")
        d_qkv = torch.full_like(qkv, float("nan"))
        F.attention_bwd(qkv, out, d_out, lse, delta, dq_acc, d_qkv, B, T, H, causal=causal)
        torch.cuda.synchronize()
        q, k, v = (qkv.view(B, T, 3, H, 64)[:, :, i].transpose(1, 2).float().requires_grad_(True) for i in range(3))
        o = torch.nn.functional.scaled_dot_product_attention(q, k, v, is_causal=causal)
        do = d_out.view(B, T, H, 64).transpose(1, 2).float()
        gq, gk, gv = torch.autograd.grad(o, (q, k, v), do)
        got = d_qkv.view(B, T, 3, H, 64)
        tag = f"B{B} T{T} H{H} causal={causal}"
        for name, i, g in (("dq", 0, gq), ("dk", 1, gk), ("dv", 2, gv)):
            # P and dS go through bf16 before the second GEMMs and dk / dv sum over up to T queries: the element-wise
            # noise floor is a few percent of the gradient's spread
            ok &= _check(f"attn bwd {name} {tag}", got[:, :, i].transpose(1, 2), g, 2e-2, rtol=5e-2, atol_scale=1.5e-1)
        ok &= _check(f"attn bwd dq_acc cleared {tag}", dq_acc, torch.zeros_like(dq_acc), 1.0, atol_scale=1.0) \
            if float(dq_acc.abs().max()) == 0.0 else False
    B, T, H = 16, 1024, 12
    C = H * 64
    qkv = _rand(B * T, 3 * C, scale=1.0)
    d_out = _rand(B * T, C, scale=1.0)
    out = torch.empty(B * T, C, device="cuda", dtype=torch.bfloat16)
    lse = torch.empty(B, H, T, device="cuda")
    F.attention_fwd(qkv, out, lse, B, T, H, causal=True)
    delta = torch.empty(B, H, T, device="cuda")
    dq_acc = torch.zeros(B * T, C, device="cuda")
    d_qkv = torch.empty_like(qkv)

    def timeit(fn, n=10):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n * 1e3

    t_ours = timeit(lambda: F.attention_bwd(qkv, out, d_out, lse, delta, dq_acc, d_qkv, B, T, H, causal=True))
    q, k, v = (qkv.view(B, T, 3, H, 64)[:, :, i].transpose(1, 2) for i in range(3))
    o4 = out.view(B, T, H, 64).transpose(1, 2)
    do4 = d_out.view(B, T, H, 64).transpose(1, 2)
    philox = torch.zeros((), dtype=torch.int64, device="cuda")
    t_lib = timeit(lambda: torch.ops.aten._scaled_dot_product_cudnn_attention_backward(
        do4, q, k, v, o4, lse.view(B, H, T, 1), philox, philox, None, None, None, T, T, 0.0, True))
    flops = 10.0 * B * H * T * T * 64 / 2
    print(f"  attention bwd B16 T1024 H12 causal: wgmma (delta + main + dq finish) {t_ours:.1f} us "
          f"({flops / t_ours / 1e6:.0f} TFLOP/s)  cuDNN SDPA backward (no gather) {t_lib:.1f} us "
          f"({flops / t_lib / 1e6:.0f} TFLOP/s)")
    return ok


def case_graph_step():
    """The CUDA-graph replay of the training step against the same step launched eagerly: same data, same schedule ->
    the same losses and parameters (up to the summation order of fp32 atomics); and the split-K reduce-add of a weight
    gradient is reproducible to fp32 round-off from run to run."""
    from ..models.gpt2 import GPT2Config, GPT2Engine
    from ..runtime.trainer import EngineTrainer, SyntheticTokens

    ok = True
    runs = {}
    for use_graph in (False, True):
        eng = GPT2Engine(GPT2Config.tiny(), 4, 128, "cuda", seed=7)
        tr = EngineTrainer(eng, lr=1e-3, use_graph=use_graph)
        data = SyntheticTokens(1000, 4, 128, n_batches=4, seed=11)
        losses = [tr.step(*data.next())]
        if not use_graph:
            # capturing runs the first step's device work twice as warm-up before the replay: do the same eagerly
            tr._device_step(); tr._device_step()
            tr.loss_host.copy_(eng.loss); torch.cuda.synchronize()
            losses[0] = float(tr.loss_host[0])
        losses += [tr.step(*data.next()) for _ in range(5)]
        torch.cuda.synchronize()
        assert use_graph == (tr.graph is not None), tr.graph_error
        runs[use_graph] = (torch.tensor(losses), eng.params.p32.clone(), eng.params.p16.float().clone())
    ok &= _check("graph vs eager: losses", runs[True][0], runs[False][0], 2e-3, rtol=5e-3, atol_scale=1e-2)
    # element-wise the weights are only comparable up to a few learning rates: where a gradient is ~0 the sign of the
    # fp32 summation noise decides the direction of Adam's (normalised) update
    ok &= _check("graph vs eager: fp32 master weights", runs[True][1], runs[False][1], 2e-3, rtol=5e-2, atol_scale=0.25)
    ok &= _check("graph vs eager: bf16 weights", runs[True][2], runs[False][2], 2e-3, rtol=5e-2, atol_scale=0.25)
    # split-K reduce-add: two runs of the same weight gradient
    Mtok, Nout, Kin = 8192, 768, 768
    dyv, x = _rand(Mtok, Nout), _rand(Mtok, Kin)
    outs = []
    for _ in range(2):
        dw = torch.zeros(Nout, Kin, device="cuda", dtype=torch.float32)
        F.gemm(dyv, x, dw, a_mn=True, b_mn=True, accumulate=True, split_k=8, block_n=512)
        torch.cuda.synchronize()
        outs.append(dw)
    ok &= _check("split-K reduce-add run-to-run", outs[0], outs[1], 1e-6, rtol=1e-5, atol_scale=1e-5)
    ok &= _check("split-K reduce-add vs fp32 reference", outs[0], dyv.float().t() @ x.float(), 1e-2)
    return ok


def case_bert_engine():
    """BERT-base-shaped MLM engine (post-LN encoder, token-type embeddings, MLM head, masked loss) vs the plain fp32
    PyTorch model on the same weights: loss and gradients; three optimizer steps reduce the loss."""
    from ..models.bert import BertConfig, BertEngine, BertReference, SyntheticMLM

    ok = True
    cfg = BertConfig.tiny()
    B, T = 4, 128
    eng = BertEngine(cfg, B, T, "cuda", seed=3)
    # break the symmetry of the zero-initialised biases / unit LayerNorm gains so that their gradients are exercised
    g = torch.Generator(device="cpu").manual_seed(9)
    for s_ in eng.params.specs:
        if len(s_.shape) == 1:
            eng.params.w32(s_.name).add_(torch.randn(s_.shape, generator=g).cuda() * 0.05)
    eng.params.w32("dec_b")[cfg.vocab_size:].zero_()
    eng.params.refresh_compute_copy()
    ref = BertReference(cfg, eng.params).cuda()
    data = SyntheticMLM(cfg.vocab_size, B, T, n_batches=1, seed=5, pin=False)
    tok, typ, lab = data.next()
    for dst, src in zip(eng.input_tensors(), (tok, typ, lab)):
        dst.copy_(src)
    assert eng.n_masked == data.n_masked
    eng.params.g32.zero_()
    eng.forward(); eng.backward()
    torch.cuda.synchronize()
    rl = ref(tok.view(B, T).cuda(), typ.view(B, T).cuda(), lab.view(B, T).cuda())
    rl.backward()
    ok &= _check("[bert] loss", eng.loss, rl.detach().reshape(1), 5e-3)
    for name in ("wte", "wpe", "wtt", "emb_ln_w", "h0.qkv_w", "h0.qkv_b", "h0.proj_w", "h0.proj_b", "h0.ln1_w", "h0.fc_w",
                 "h0.fc_b", "h0.fc2_w", "h0.fc2_b", "h1.ln2_b", "h1.fc2_w", "mlm_w", "mlm_b", "mlm_ln_w", "dec_b"):
        gref = ref.p(name).grad
        got = eng.params.grad(name)
        if name == "dec_b":
            gref, got = gref[:cfg.vocab_size], got[:cfg.vocab_size]
        ok &= _check(f"[bert] grad {name}", got, gref, 4e-2, rtol=1e-1, atol_scale=2.5e-1)
    l0 = float(eng.loss.item())
    for step in range(1, 4):
        eng.optimizer_step(lr=1e-3, step=step)
        eng.forward(); eng.backward()
    l1 = float(eng.loss.item())
    print(f"  [bert] loss {l0:.4f} -> {l1:.4f}")
    ok &= l1 < l0
    return ok


# ----------------------------------------------------------------------------- attention
def case_attention():
    """wgmma flash-attention forward vs. an fp32 PyTorch reference (causal and full), plus its device time next to
    the cuDNN SDPA kernel PyTorch dispatches to."""
    ok = True
    for (B, T, H, causal) in [(2, 256, 3, True), (1, 128, 2, True), (2, 384, 2, False), (2, 1024, 12, True),
                              (1, 512, 2, "ramp"), (1, 512, 2, "ramp-full")]:
        C = H * 64
        qkv = _rand(B * T, 3 * C, scale=1.0)
        if isinstance(causal, str):
            # adversarial: later keys score enormously higher than earlier ones (logit blow-up), which forces the
            # kernel's lagging softmax reference through its exact-redo path
            qv = qkv.view(B, T, 3, H, 64)
            ramp = torch.linspace(0.0, 40.0, T, device="cuda").view(1, T, 1, 1)
            qv[:, :, 1] = (qv[:, :, 1].float() + ramp * qv[:, :1, 0].float().sign()).bfloat16()
            qv[:, :, 0] = qv[:, :1, 0].abs() * 4 + 0.0 * qv[:, :, 0]
            causal = causal == "ramp"
        out = torch.empty(B * T, C, device="cuda", dtype=torch.bfloat16)
        lse = torch.empty(B, H, T, device="cuda")
        F.attention_fwd(qkv, out, lse, B, T, H, causal=causal)
        q, k, v = (qkv.view(B, T, 3, H, 64)[:, :, i].transpose(1, 2).float() for i in range(3))
        s = (q @ k.transpose(-1, -2)) * 0.125
        if causal:
            s = s.masked_fill(torch.ones(T, T, device="cuda", dtype=torch.bool).triu(1), float("-inf"))
        ref = (torch.softmax(s, -1) @ v).transpose(1, 2).reshape(B * T, C)
        ok &= _check(f"attn fwd out B{B} T{T} H{H} causal={causal}", out, ref, 2e-2, atol_scale=5e-2)
        ok &= _check(f"attn fwd lse B{B} T{T} H{H} causal={causal}", lse, torch.logsumexp(s, -1), 1e-3)
    # timing at the GPT-2 small shape
    B, T, H = 16, 1024, 12
    C = H * 64
    qkv = _rand(B * T, 3 * C, scale=1.0)
    out = torch.empty(B * T, C, device="cuda", dtype=torch.bfloat16)
    lse = torch.empty(B, H, T, device="cuda")

    def timeit(fn, n=20):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n * 1e3

    t_ours = timeit(lambda: F.attention_fwd(qkv, out, lse, B, T, H, causal=True))
    q, k, v = (qkv.view(B, T, 3, H, 64)[:, :, i].transpose(1, 2) for i in range(3))
    t_lib = timeit(lambda: torch.nn.functional.scaled_dot_product_attention(q, k, v, is_causal=True))
    flops = 4.0 * B * H * T * T * 64 / 2
    print(f"  attention fwd B16 T1024 H12 causal: wgmma {t_ours:.1f} us ({flops / t_ours / 1e6:.0f} TFLOP/s)  "
          f"cuDNN SDPA {t_lib:.1f} us ({flops / t_lib / 1e6:.0f} TFLOP/s)")
    return ok


# ----------------------------------------------------------------------------- document-masked attention
def doc_start_from_lengths(lengths, T):
    """int32 [T] document starts of one sequence cut into documents of the given lengths (cycled until T is filled)."""
    ds, pos, i = [], 0, 0
    while pos < T:
        n = min(lengths[i % len(lengths)], T - pos)
        ds += [pos] * n
        pos += n
        i += 1
    return torch.tensor(ds, dtype=torch.int32)


def _doc_mask_ref(qkv, d_out, B, T, H, doc_start):
    """fp32 attention with the explicit boolean document mask: out, lse, and dq / dk / dv for ``d_out``."""
    q, k, v = (qkv.view(B, T, 3, H, 64)[:, :, i].transpose(1, 2).float().requires_grad_(True) for i in range(3))
    ds = doc_start.view(B, 1, T, 1).long()
    kk = torch.arange(T, device=qkv.device).view(1, 1, 1, T)
    qq = torch.arange(T, device=qkv.device).view(1, 1, T, 1)
    allowed = (kk >= ds) & (kk <= qq)
    s = ((q @ k.transpose(-1, -2)) * 0.125).masked_fill(~allowed, float("-inf"))
    o = torch.softmax(s, -1) @ v
    grads = torch.autograd.grad(o, (q, k, v), d_out.view(B, T, H, 64).transpose(1, 2).float())
    return (o.detach().transpose(1, 2).reshape(B * T, H * 64), torch.logsumexp(s.detach(), -1), grads)


def _run_attn(qkv, d_out, B, T, H, doc_start):
    C = H * 64
    out = torch.empty(B * T, C, device="cuda", dtype=torch.bfloat16)
    lse = torch.empty(B, H, T, device="cuda")
    F.attention_fwd(qkv, out, lse, B, T, H, causal=True, doc_start=doc_start)
    delta = torch.empty(B, H, T, device="cuda")
    dq_acc = torch.zeros(B * T, C, device="cuda")
    d_qkv = torch.full_like(qkv, float("nan"))
    F.attention_bwd(qkv, out, d_out, lse, delta, dq_acc, d_qkv, B, T, H, causal=True, doc_start=doc_start)
    torch.cuda.synchronize()
    return out, lse, d_qkv, dq_acc


def case_attention_docs():
    """Document-masked wgmma attention forward and backward vs an fp32 reference with an explicit boolean mask, on
    layouts that put document boundaries everywhere a block edge could go wrong; one document per row against the
    unmasked causal kernels; every token its own document."""
    ok = True
    mixed = [1, 63, 64, 65, 127, 128, 129]
    layouts = [
        (1, 128, 1, [[1, 63, 64]]),
        (1, 256, 3, [mixed]),
        (1, 1024, 12, [mixed]),
        (1, 256, 1, [[127, 129]]),                     # a document starting at the last row of the first 128-row tile
        (2, 256, 3, [[255, 1], [64, 64, 1, 127]]),     # ... and of the second; B = 2 with a different layout per row
        (2, 1024, 3, [mixed[::-1], [300, 700, 24]]),
        (1, 128, 3, [[1]]),                            # every token its own document
    ]
    for B, T, H, per_row in layouts:
        ds = torch.cat([doc_start_from_lengths(per_row[b % len(per_row)], T) for b in range(B)]).cuda()
        C = H * 64
        qkv = _rand(B * T, 3 * C)
        d_out = _rand(B * T, C)
        out, lse, d_qkv, dq_acc = _run_attn(qkv, d_out, B, T, H, ds)
        ref_o, ref_lse, (gq, gk, gv) = _doc_mask_ref(qkv, d_out, B, T, H, ds)
        tag = f"B{B} T{T} H{H} docs={per_row}"[:80]
        ok &= _check(f"doc attn fwd out {tag}", out, ref_o, 2e-2, atol_scale=5e-2)
        ok &= _check(f"doc attn fwd lse {tag}", lse, ref_lse, 1e-3)
        got = d_qkv.view(B, T, 3, H, 64)
        for name, i, g in (("dq", 0, gq), ("dk", 1, gk), ("dv", 2, gv)):
            if per_row == [[1]] and i < 2:
                # a row that sees only itself has P = 1 and o = v, so dS = P (dP - delta) is exactly 0: dq and dk are 0 up
                # to the rounding of dP and delta (dO . v in the tensor cores vs dO . bf16(o)), against O(1) gradients
                worst = float(got[:, :, i].abs().max())
                print(f"  own-document rows: |{name}| <= {worst:.2e} (exactly 0 in exact arithmetic)")
                ok &= worst < 1e-5
                continue
            ok &= _check(f"doc attn bwd {name} {tag}", got[:, :, i].transpose(1, 2), g, 2e-2, rtol=5e-2,
                         atol_scale=1.5e-1)
        ok &= float(dq_acc.abs().max()) == 0.0
        if per_row == [[1]]:
            # each row attends to itself only: out is that row's v, lse its own scaled score
            v = qkv.view(B, T, 3, H, 64)[:, :, 2].reshape(B * T, C)
            same = bool(torch.equal(out, v))
            print(f"  own-document rows: out == v bit for bit: {same}")
            ok &= same
            q, k = (qkv.view(B, T, 3, H, 64)[:, :, i].float() for i in range(2))
            ok &= _check("own-document lse = own scaled score", lse, ((q * k).sum(-1) * 0.125).permute(0, 2, 1), 1e-4)
    # one document per row: the masked kernels visit the same blocks in the same order as the causal ones
    B, T, H = 2, 1024, 12
    qkv = _rand(B * T, 3 * H * 64)
    d_out = _rand(B * T, H * 64)
    ref = _run_attn(qkv, d_out, B, T, H, None)
    got = _run_attn(qkv, d_out, B, T, H, torch.zeros(B * T, dtype=torch.int32, device="cuda"))
    for name, a, b in (("out", got[0], ref[0]), ("lse", got[1], ref[1]),
                       ("dk", got[2].view(B * T, 3, -1)[:, 1], ref[2].view(B * T, 3, -1)[:, 1]),
                       ("dv", got[2].view(B * T, 3, -1)[:, 2], ref[2].view(B * T, 3, -1)[:, 2])):
        same = bool(torch.equal(a, b))
        print(f"  one document per row vs causal kernel: {name} bit-identical: {same}")
        ok &= same
    # dq is summed over key blocks with fp32 atomics, whose order differs from run to run in either kernel
    dq_g, dq_r = got[2].view(B * T, 3, -1)[:, 0], ref[2].view(B * T, 3, -1)[:, 0]
    ok &= _check("one document per row vs causal kernel: dq (atomic order)", dq_g, dq_r, 1e-3, rtol=1e-2,
                 atol_scale=1e-2)
    # unsupported: a mask with full (non-causal) attention is refused by the entry point and by the kernel
    try:
        F.attention_fwd(qkv, got[0], got[1], B, T, H, causal=False, doc_start=torch.zeros(B * T, dtype=torch.int32,
                                                                                          device="cuda"))
        ok = False
    except ValueError:
        pass
    rc = F.lib.load().aitj_attn_fwd(qkv.data_ptr(), got[0].data_ptr(), got[1].data_ptr(), got[1].data_ptr(), B, T, H,
                                    0, 0.0, torch.cuda.current_stream().cuda_stream)
    ok &= rc == -5
    return ok


def _doc_tokens(B, T, vocab, eot, lengths, seed):
    """Token ids with documents of the given lengths (each opened by ``eot``, as in llm.c shards)."""
    g = torch.Generator().manual_seed(seed)
    tok = torch.randint(0, vocab - 1, (B, T), generator=g)
    tok[tok == eot] = 0
    ds = torch.stack([doc_start_from_lengths(lengths[b % len(lengths)], T) for b in range(B)])
    starts = ds == torch.arange(T)
    starts[:, 0] = False
    tok[starts] = eot
    return tok, ds


def case_gpt2_docs():
    """GPT2Engine(doc_mask=True) vs GPT2Reference with the same boolean document mask (loss, gradients), and documents
    that cannot see each other: changing one document leaves every per-token loss of the others bit-identical."""
    from ..models.gpt2 import GPT2Config, GPT2Engine, GPT2Reference

    ok = True
    cfg = GPT2Config(vocab_size=1000, n_layer=2, n_head=4, n_embd=256, block_size=256, name="t")
    B, T, eot = 4, 256, 999
    eng = GPT2Engine(cfg, B, T, "cuda", seed=3, doc_mask=True)
    assert eng.attn_impl == "wgmma" and eng.attn_bwd_impl == "wgmma"
    ref = GPT2Reference(cfg, eng.params).cuda()
    tok, ds = _doc_tokens(B, T, cfg.vocab_size, eot, [[40, 1, 100, 115], [256], [7, 64, 129, 56], [1]], 5)
    tok, ds = tok.cuda(), ds.cuda()
    tgt = torch.roll(tok, -1, dims=1)
    for dst, src in zip(eng.input_tensors(), (tok, tgt, ds)):
        dst.copy_(src.reshape(-1))
    eng.params.g32.zero_()
    eng.forward(); eng.backward()
    torch.cuda.synchronize()
    rl = ref(tok, tgt, ds)
    rl.backward()
    ok &= _check("[doc_mask] loss", eng.loss, rl.detach().reshape(1), 5e-3)
    for name in ("wte", "wpe", "h0.qkv_w", "h0.qkv_b", "h0.proj_w", "h0.fc_w", "h0.fc_b", "h0.fc2_w", "h1.ln1_w",
                 "h1.ln2_b", "h1.fc2_w", "lnf_w", "lnf_b"):
        ok &= _check(f"[doc_mask] grad {name}", eng.params.grad(name), ref.p(name).grad, 4e-2, rtol=1e-1,
                     atol_scale=2.5e-1)
    # isolation: row 0's third document ([41, 141)) gets new tokens (its end-of-text opener stays)
    for masked in (True, False):
        e = eng if masked else GPT2Engine(cfg, B, T, "cuda", seed=3)
        losses = []
        for variant in range(2):
            t = tok.clone()
            if variant:
                t[0, 42:141] = (t[0, 42:141] + 17) % (cfg.vocab_size - 1)
            ins = (t, torch.roll(t, -1, dims=1), ds)
            for dst, src in zip(e.input_tensors(), ins):
                dst.copy_(src.reshape(-1))
            e.forward()
            torch.cuda.synchronize()
            losses.append(e.losses.view(B, T).clone())
        others = torch.ones(B, T, dtype=torch.bool, device="cuda")
        others[0, 41:141] = False
        same = bool(torch.equal(losses[0][others], losses[1][others]))
        later_changed = not torch.equal(losses[0][0, 141:], losses[1][0, 141:])
        print(f"  doc_mask={masked}: losses of the other documents bit-identical after changing one: {same}; "
              f"later documents of that row changed: {later_changed}")
        ok &= same if masked else later_changed
    # three optimizer steps reduce the loss
    for dst, src in zip(eng.input_tensors(), (tok, tgt, ds)):
        dst.copy_(src.reshape(-1))
    eng.params.g32.zero_()
    eng.forward(); eng.backward()
    l0 = float(eng.loss.item())
    for step in range(1, 4):
        eng.optimizer_step(lr=1e-3, step=step)
        eng.forward(); eng.backward()
    l1 = float(eng.loss.item())
    print(f"  [doc_mask] loss {l0:.4f} -> {l1:.4f}")
    ok &= l1 < l0
    return ok


CASES = {
    "attention": case_attention,
    "attention_docs": case_attention_docs,
    "gpt2_docs": case_gpt2_docs,
    "gemm_2cta": case_gemm_2cta,
    "gemm_quad": case_gemm_quad,
    "graph_step": case_graph_step,
    "bert_engine": case_bert_engine,
    "attention_bwd": case_attention_bwd,
    "gpt2_engine": case_gpt2_engine,
    "gemm_tn": case_gemm_tn,
    "gemm_nn": case_gemm_nn,
    "gemm_tt": case_gemm_tt,
    "gemm_epilogue": case_gemm_epilogue,
    "fused_ops": case_fused_ops,
}


def main(argv=None) -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--case", default="all")
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        print("no CUDA device", file=sys.stderr)
        return 2
    torch.manual_seed(1234)
    names = list(CASES) if args.case == "all" else [args.case]
    ok = True
    for n in names:
        print(f"[selfcheck] {n}", flush=True)
        t0 = time.time()
        try:
            r = CASES[n]()
        except Exception as e:  # noqa: BLE001
            print(f"  EXCEPTION {type(e).__name__}: {e}", flush=True)
            r = False
        print(f"[selfcheck] {n}: {'PASS' if r else 'FAIL'} ({time.time() - t0:.1f}s)", flush=True)
        ok &= bool(r)
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
