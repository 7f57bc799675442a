"""GPT-2 medium, large and XL: the model table, the wide LayerNorm kernels (``ops/csrc/layernorm_wide.cu``) and the
engine's choice of LayerNorm kernel by width.

On the CPU the engines run with the kernel entry points emulated (``tests/kernel_emulation.py``) at each new width, one
layer deep, against the fp32 reference model; the GEMM stand-in refuses any GEMM the built library has no kernel for.
On the H100 the wide kernels are checked against fp64, the engines against the reference at full width, and every size
trains a few steps at full depth.
"""
import math
import os
import re
import sys

import pytest
import torch
import yaml

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import kernel_emulation as ke  # noqa: E402
from trainingjob_operator_b200.models.gpt2 import GPT2_MODELS, GPT2Config, gpt2_config, gpt2_param_specs  # noqa: E402
from trainingjob_operator_b200.ops import functional as F  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------------------------ the model table
@pytest.mark.parametrize("name,layers,heads,width,unpadded", [
    ("gpt2", 12, 12, 768, 124_439_808),
    ("gpt2-medium", 24, 16, 1024, 354_823_168),
    ("gpt2-large", 36, 20, 1280, 774_030_080),
    ("gpt2-xl", 48, 25, 1600, 1_557_611_200),
])
def test_the_table_has_gpt2s_shapes_and_parameter_counts(name, layers, heads, width, unpadded):
    cfg = gpt2_config(name)
    assert (cfg.n_layer, cfg.n_head, cfg.n_embd, cfg.vocab_size, cfg.padded_vocab, cfg.block_size) == \
        (layers, heads, width, 50257, 50304, 1024)
    assert cfg.n_embd // cfg.n_head == 64
    padded = sum(math.prod(s.shape) for s in gpt2_param_specs(cfg))
    assert padded - (cfg.padded_vocab - cfg.vocab_size) * width == unpadded
    if name == "gpt2":
        assert padded == 124_475_904
    assert cfg is not GPT2_MODELS[name] and cfg == GPT2_MODELS[name]      # a copy: callers cannot edit the table


def test_the_table_keeps_small_and_tiny_as_they_were():
    assert gpt2_config("gpt2") == GPT2Config.small() and gpt2_config("gpt2-tiny") == GPT2Config.tiny()


# ------------------------------------------------------------------------------------ stand-ins of the wide pair
# CPU stand-ins of ``F.layernorm_wide_fwd`` / ``F.layernorm_wide_bwd`` in the manner of ``kernel_emulation``: the
# wrappers' own checks first, then the same in-place outputs and accumulations with fp32 math.
def layernorm_wide_fwd(x, gamma, beta, y, mean, rstd, eps=1e-5):
    ke.CALLS["n"] += 1
    F.check_layernorm_wide_fwd(x, gamma, beta, y, mean, rstd, eps)
    xf = x.float()
    mu = xf.mean(1)
    r = torch.rsqrt(xf.var(1, unbiased=False) + eps)
    mean.copy_(mu)
    rstd.copy_(r)
    y.copy_((xf - mu[:, None]) * r[:, None] * gamma.float() + beta.float())
    return y


def layernorm_wide_bwd(dy, x, gamma, mean, rstd, dx, dgamma, dbeta, dres=None, dxsum=None):
    ke.CALLS["n"] += 1
    F.check_layernorm_wide_bwd(dy, x, gamma, mean, rstd, dx, dgamma, dbeta, dres, dxsum)
    h = (x.float() - mean[:, None]) * rstd[:, None]
    d = dy.float()
    ke._dst(dgamma).add_((d * h).sum(0))
    ke._dst(dbeta).add_(d.sum(0))
    a = d * gamma.float()
    v = rstd[:, None] * (a - a.mean(1, keepdim=True) - h * (a * h).mean(1, keepdim=True))
    if dres is not None:
        v = v + dres.float()
    if dxsum is not None:
        ke._dst(dxsum).add_(v.sum(0))
    dx.copy_(v)                     # after the reads: dx may alias dres / dy
    return dx


def install(monkeypatch):
    """``kernel_emulation.install`` plus the stand-ins of the wide LayerNorm pair."""
    ke.install(monkeypatch)
    monkeypatch.setattr(F, "layernorm_wide_fwd", layernorm_wide_fwd)
    monkeypatch.setattr(F, "layernorm_wide_bwd", layernorm_wide_bwd)


# ------------------------------------------------------------------------------------ emulated engines
def _ln_calls(monkeypatch):
    """Names of the LayerNorm entry points the engine calls, in order."""
    seen = []
    for name in ("layernorm_fwd", "layernorm_bwd", "layernorm_wide_fwd", "layernorm_wide_bwd"):
        fn = getattr(F, name)

        def wrapped(*a, _fn=fn, _name=name, **k):
            seen.append(_name)
            return _fn(*a, **k)

        monkeypatch.setattr(F, name, wrapped)
    return seen


def rel(a, b):
    return float((a.float() - b.float()).norm() / (b.float().norm() + 1e-12))


@pytest.mark.parametrize("width,impl", [(1024, "wide"), (1280, "wide"), (1600, "wide"), (768, "fused")])
def test_emulated_engine_at_each_width_matches_the_reference(monkeypatch, width, impl):
    """Forward, backward and an optimizer step at a GPT-2 width, one layer and T = 128: the loss and every gradient
    slice against ``GPT2Reference``, the LayerNorm launches on the kernels the engine chose for the width, and every
    GEMM on a compiled kernel (the GEMM stand-in raises the library's "no kernel" refusal otherwise)."""
    from trainingjob_operator_b200.models.gpt2 import GPT2Engine, GPT2Reference

    install(monkeypatch)
    seen = _ln_calls(monkeypatch)
    cfg = GPT2Config(vocab_size=512, n_layer=1, n_head=width // 64, n_embd=width, block_size=128, name="t")
    B, T = 1, 128
    eng = GPT2Engine(cfg, B, T, "cpu", seed=3)
    assert eng.ln_impl == impl
    g = torch.Generator().manual_seed(9)
    for s in eng.params.specs:               # LayerNorm gains and biases away from their symmetric initial values
        if len(s.shape) == 1:
            eng.params.w32(s.name).add_(torch.randn(s.shape, generator=g) * 0.05)
    eng.params.refresh_compute_copy()
    ref = GPT2Reference(cfg, eng.params)
    tok = torch.randint(0, cfg.vocab_size, (B, T), generator=torch.Generator().manual_seed(5))
    tgt = torch.roll(tok, -1, dims=1)
    eng.tok.copy_(tok.view(-1))
    eng.tgt.copy_(tgt.view(-1))
    eng.params.g32.zero_()
    eng.forward()
    eng.backward()
    want = {"fused": {"layernorm_fwd", "layernorm_bwd"}, "wide": {"layernorm_wide_fwd", "layernorm_wide_bwd"}}[impl]
    assert set(seen) == want and len(seen) == 6, seen          # ln1, ln2, lnf: forward and backward
    loss = ref(tok, tgt)
    loss.backward()
    assert abs(float(eng.loss) - float(loss.detach())) < 2e-2 * float(loss.detach())
    for name in ("wte", "wpe", "h0.qkv_w", "h0.qkv_b", "h0.proj_w", "h0.proj_b", "h0.fc_w", "h0.fc_b", "h0.fc2_w",
                 "h0.fc2_b", "h0.ln1_w", "h0.ln1_b", "h0.ln2_w", "h0.ln2_b", "lnf_w", "lnf_b"):
        assert rel(eng.params.grad(name), ref.p(name).grad) < 6e-2, name
    before = eng.params.w32("h0.ln1_w").clone()
    eng.optimizer_step(lr=1e-3, step=1)
    assert not torch.equal(eng.params.w32("h0.ln1_w"), before)
    assert torch.equal(eng.params.p16, eng.params.p32.to(torch.bfloat16))
    assert float(eng.params.g32.abs().max()) == 0.0


@pytest.mark.parametrize("width", [1004, 2056, 4])
def test_an_engine_of_a_width_no_layernorm_kernel_serves_is_refused(width):
    from trainingjob_operator_b200.models.gpt2 import GPT2Engine

    cfg = GPT2Config(vocab_size=512, n_layer=1, n_head=1, n_embd=width, block_size=128, name="t")
    with pytest.raises(ValueError, match=f"no LayerNorm kernel serves n_embd={width}"):
        GPT2Engine(cfg, 1, 128, "cpu")


def _ln_args(M, C, dres=True, dxsum=True):
    bf, f32 = dict(dtype=torch.bfloat16), dict(dtype=torch.float32)
    return dict(dy=torch.zeros(M, C, **bf), x=torch.zeros(M, C, **bf), gamma=torch.zeros(C, **bf),
                mean=torch.zeros(M, **f32), rstd=torch.zeros(M, **f32), dx=torch.zeros(M, C, **bf),
                dgamma=torch.zeros(C, **f32), dbeta=torch.zeros(C, **f32),
                dres=torch.zeros(M, C, **bf) if dres else None, dxsum=torch.zeros(C, **f32) if dxsum else None)


# (edit of a valid call, the error, whether the forward takes the edited argument too)
BAD_WIDE_CALLS = [
    (lambda a: a.update(x=torch.zeros(4, 1004, dtype=torch.bfloat16)), "multiple of 8", True),
    (lambda a: a.update(x=torch.zeros(4, 2056, dtype=torch.bfloat16)), "multiple of 8 in [8, 2048]", True),
    (lambda a: a.update(x=a["x"].float()), "x must be torch.bfloat16", True),
    (lambda a: a.update(x=torch.zeros(8, 1600, dtype=torch.bfloat16)[::2]), "x must be contiguous", True),
    (lambda a: a.update(gamma=torch.zeros(1280, dtype=torch.bfloat16)), "gamma must hold 1600", True),
    (lambda a: a.update(mean=torch.zeros(3)), "mean must hold 4", True),
    (lambda a: a.update(dy=torch.zeros(4, 1280, dtype=torch.bfloat16)), "dy must be [4, 1600]", False),
    (lambda a: a.update(dres=torch.zeros(5, 1600, dtype=torch.bfloat16)), "dres must be [4, 1600]", False),
    (lambda a: a.update(dx=torch.zeros(4 * 1600 + 8, dtype=torch.bfloat16)[1:4 * 1600 + 1].view(4, 1600)),
     "dx must be 16-byte aligned", False),
    (lambda a: a.update(dgamma=torch.zeros(1280)), "dgamma must be an fp32 gradient of shape (1600,)", False),
    (lambda a: a.update(dxsum=torch.zeros(1600, dtype=torch.float64)), "dxsum must be an fp32 gradient", False),
    (lambda a: a.update(dbeta=F.PeerView(torch.zeros(1600))), "must all be local, all multicast or all owner-sharded",
     False),
]


@pytest.mark.parametrize("i", range(len(BAD_WIDE_CALLS)), ids=[c[1] for c in BAD_WIDE_CALLS])
def test_the_wide_layernorm_wrappers_and_stand_ins_refuse_alike(i):
    """The wide entry points refuse nothing themselves: their wrappers check every argument, and the stand-ins apply
    the same checks."""
    edit, what, fwd_too = BAD_WIDE_CALLS[i]
    args = _ln_args(4, 1600)
    edit(args)
    for fn in (F.layernorm_wide_bwd, layernorm_wide_bwd):
        with pytest.raises(ValueError, match=re.escape(what)):
            fn(**args)
    if fwd_too:
        fwd = dict(x=args["x"], gamma=args["gamma"], beta=args["gamma"], y=torch.zeros_like(args["x"]),
                   mean=args["mean"], rstd=args["rstd"])
        for fn in (F.layernorm_wide_fwd, layernorm_wide_fwd):
            with pytest.raises(ValueError, match=re.escape(what)):
                fn(**fwd)


def test_the_wide_stand_ins_accept_every_width_up_to_2048():
    for C in (8, 1024, 1280, 1600, 2048):
        a = _ln_args(3, C)
        layernorm_wide_fwd(a["x"], a["gamma"], a["gamma"], torch.zeros_like(a["x"]), a["mean"], a["rstd"])
        layernorm_wide_bwd(**a)


# ------------------------------------------------------------------------------------ worker and CLI
@pytest.mark.parametrize("model", ["gpt2-medium", "gpt2-large", "gpt2-xl"])
def test_the_worker_and_generate_cli_take_the_new_names(model):
    from trainingjob_operator_b200.cmd import generate
    from trainingjob_operator_b200.runtime.worker import parse_args

    a = parse_args(["--model", model, "--batch", "4", "--global-batch", "64", "--data", "d.bin", "--doc-mask",
                    "--eval-data", "v.bin", "--eval-every", "10", "--generate-every", "50", "--ckpt-every", "100"])
    assert a.model == model and a.generate_prompt == [50256] and a.doc_mask and a.global_batch == 64
    assert generate.parse_args(["--model", model, "--ckpt", "c.pt"]).model == model


@pytest.mark.parametrize("argv,what", [
    (["--model", "gpt2-xl", "--data", "d.bin", "--doc-mask", "--eot-token", "50257"],
     "--eot-token 50257 is outside the vocabulary of gpt2-xl (size 50257)"),
    (["--model", "gpt2-large", "--generate-every", "2", "--generate-tokens", "1024"],
     "exceed the block size of gpt2-large (1024)"),
    (["--model", "gpt2-medium", "--generate-every", "2", "--top-k", "50258"],
     "--top-k 50258 exceeds the vocabulary of gpt2-medium (size 50257)"),
    (["--model", "gpt2-xl", "--eval-data", "v.bin", "--gemm", "cublas"], "--eval-data needs --gemm wgmma"),
    (["--model", "gpt2-xl", "--batch", "8", "--global-batch", "12"], "is not a multiple of --batch 8"),
    (["--model", "bert", "--data", "d.bin"], "--data trains GPT-2 models only, not bert"),
    (["--model", "gpt2-xxl"], "invalid choice: 'gpt2-xxl'"),
])
def test_the_worker_refuses_bad_combinations_with_its_messages(capsys, argv, what):
    from trainingjob_operator_b200.runtime.worker import parse_args

    with pytest.raises(SystemExit):
        parse_args(argv)
    assert what in capsys.readouterr().err


def test_a_checkpoint_of_another_size_is_refused(monkeypatch, tmp_path):
    from trainingjob_operator_b200.cmd import generate
    from trainingjob_operator_b200.runtime.checkpoint import load_into

    install(monkeypatch)
    monkeypatch.setitem(GPT2_MODELS, "gpt2-medium", GPT2Config(vocab_size=512, n_layer=1, n_head=16, n_embd=1024,
                                                               block_size=128, name="gpt2-medium"))
    from trainingjob_operator_b200.models.gpt2 import GPT2Engine

    other = GPT2Engine(GPT2Config(vocab_size=512, n_layer=1, n_head=20, n_embd=1280, block_size=128, name="t"), 1, 1,
                       "cpu")
    path = str(tmp_path / "ck.pt")
    torch.save({"step": 1, "state": [t.cpu() for t in other.params.state_tensors()]}, path)
    with pytest.raises(ValueError, match="does not match the model"):
        generate.main(["--model", "gpt2-medium", "--ckpt", path, "--cpu", "--tokens", "1", "--count", "1"])
    assert load_into(path, other.params.state_tensors()) is not None


def test_the_xl_example_validates_and_its_worker_arguments_parse():
    from trainingjob_operator_b200.api.validation import validate_dict
    from trainingjob_operator_b200.runtime.worker import parse_args

    d = yaml.safe_load(open(os.path.join(ROOT, "examples", "gpt2-xl-8gpu.yaml")))
    assert validate_dict(d) == []
    trainer = d["spec"]["replicaSpecs"]["trainer"]
    assert trainer["replicas"] == 8
    argv = trainer["template"]["spec"]["containers"][0]["args"]
    a = parse_args(argv[argv.index("trainingjob_operator_b200.runtime.worker") + 1:])
    assert a.model == "gpt2-xl" and a.global_batch % a.batch == 0 and a.ckpt_every > 0


# ------------------------------------------------------------------------------------ GPU
def _rand(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, device="cuda", generator=g) * scale).bfloat16()


def _close(name, got, ref, atol, rtol):
    got, ref = got.double(), ref.double()
    bad = (got - ref).abs() > atol + rtol * ref.abs()
    assert torch.isfinite(got).all(), name
    assert not bad.any(), (f"{name}: {int(bad.sum())} of {ref.numel()} outside, first at {bad.nonzero()[0].tolist()}, "
                           f"worst {float((got - ref).abs().max()):.3g}")


@pytest.mark.gpu
@pytest.mark.parametrize("C", [1280, 1600, 1024, 8, 2048])
@pytest.mark.parametrize("M", [1, 77, 4099])
def test_wide_layernorm_kernels_against_fp64(C, M):
    """Forward and backward of the wide kernels against fp64 on the same bf16 inputs, M not a multiple of the 8 rows a
    block takes at a time, with and without dres / dxsum.  The parameter gradients are added into slices of one flat
    buffer that starts at 1000 + noise, so a store outside its slice, or an overwrite instead of an add, shows."""
    x = _rand(M, C, scale=2.0, seed=1) + 0.5
    gamma, beta = _rand(C, seed=2) * 0.5 + 1.0, _rand(C, seed=3) * 0.1
    y = torch.full_like(x, float("nan"))
    mean, rstd = torch.full((M,), float("nan"), device="cuda"), torch.full((M,), float("nan"), device="cuda")
    F.layernorm_wide_fwd(x, gamma, beta, y, mean, rstd)
    xd = x.double()
    mu = xd.mean(1, keepdim=True)
    rs = torch.rsqrt(xd.var(1, unbiased=False, keepdim=True) + 1e-5)
    h = (xd - mu) * rs
    _close("mean", mean, mu[:, 0], 1e-6, 1e-5)
    _close("rstd", rstd, rs[:, 0], 0, 1e-4)
    _close("y", y, h * gamma.double() + beta.double(), 1e-2, 2 ** -7)
    dy = _rand(M, C, seed=4)
    for with_res, with_xsum in ((True, True), (False, False), (True, False), (False, True)):
        guard = 64
        gen = torch.Generator(device="cuda").manual_seed(6)
        flat = 1000 + torch.rand(3 * C + 4 * guard, device="cuda", generator=gen)
        start = flat.clone()
        sl = [slice(guard + i * (C + guard), guard + i * (C + guard) + C) for i in range(3)]
        dres = _rand(M, C, seed=5) if with_res else None
        dx = torch.full_like(x, float("nan"))
        F.layernorm_wide_bwd(dy, x, gamma, mean, rstd, dx, flat[sl[0]], flat[sl[1]], dres=dres,
                             dxsum=flat[sl[2]] if with_xsum else None)
        torch.cuda.synchronize()
        a = dy.double() * gamma.double()
        want = rs * (a - a.mean(1, keepdim=True) - h * (a * h).mean(1, keepdim=True))
        if with_res:
            want = want + dres.double()
        _close("dx", dx, want, 2e-2 * float(want.std()), 2 ** -7)
        for k, (s, term) in enumerate(((sl[0], dy.double() * h), (sl[1], dy.double()), (sl[2], want))):
            if k == 2 and not with_xsum:
                _close("dxsum untouched", flat[s], start[s], 0, 0)
                continue
            bound = 1e-5 * term.abs().sum(0) + 1e-3
            _close(f"param grad {k}", flat[s] - start[s], term.sum(0), bound, 0)
        mask = torch.ones_like(flat, dtype=torch.bool)
        for s in sl:
            mask[s] = False
        assert torch.equal(flat[mask], start[mask]), "a parameter gradient landed outside its slice"


@pytest.mark.gpu
@pytest.mark.parametrize("M", [77, 16384])
def test_wide_and_fused_layernorm_agree_at_1024(M):
    C = 1024
    x, dy, dres = _rand(M, C, seed=1), _rand(M, C, seed=2), _rand(M, C, seed=3)
    gamma, beta = _rand(C, seed=4) * 0.5 + 1, _rand(C, seed=5)
    outs = []
    for fwd, bwd in ((F.layernorm_fwd, F.layernorm_bwd), (F.layernorm_wide_fwd, F.layernorm_wide_bwd)):
        y, mean, rstd = torch.empty_like(x), torch.empty(M, device="cuda"), torch.empty(M, device="cuda")
        fwd(x, gamma, beta, y, mean, rstd)
        dx, g = torch.empty_like(x), torch.zeros(3, C, device="cuda")
        bwd(dy, x, gamma, mean, rstd, dx, g[0], g[1], dres=dres, dxsum=g[2])
        outs.append((y, mean, rstd, dx, g))
    torch.cuda.synchronize()
    (y0, m0, r0, dx0, g0), (y1, m1, r1, dx1, g1) = outs
    _close("y", y1, y0, 1e-2, 2 ** -7)
    _close("mean", m1, m0, 1e-6, 1e-5)
    _close("rstd", r1, r0, 0, 1e-5)
    _close("dx", dx1, dx0, 1e-2, 2 ** -7)
    _close("dgamma, dbeta, dxsum", g1, g0, 1e-3 * float(g0.abs().max()), 1e-4)


def _gpu_engine(C, layers=2, B=2, T=256, doc_mask=False, env=None, seed=3, vocab=50257):
    from trainingjob_operator_b200.models.gpt2 import GPT2Engine

    old = {k: os.environ.pop(k, None) for k in ("AITJ_ATTN", "AITJ_ATTN_BWD")}
    os.environ.update(env or {})
    try:
        cfg = GPT2Config(vocab_size=vocab, n_layer=layers, n_head=C // 64, n_embd=C, name=f"w{C}")
        eng = GPT2Engine(cfg, B, T, "cuda", seed=seed, doc_mask=doc_mask)
    finally:
        for k, v in old.items():
            os.environ.pop(k, None)
            if v is not None:
                os.environ[k] = v
    return cfg, eng


@pytest.mark.gpu
@pytest.mark.parametrize("C", [1024, 1280, 1600])
@pytest.mark.parametrize("variant", ["cudnn", "wgmma-attention", "doc-mask"])
def test_engine_at_full_width_against_the_reference(C, variant):
    """Two layers at each new width, loss and gradients against the fp32 model within ``case_gpt2_engine``'s bounds, at
    its vocabulary of 1000: with 50257 rows and 512 tokens, most rows of the wte gradient hold only the tiny logit
    terms, and the element-wise bound, tied to the spread of the whole gradient, becomes tighter than bf16 allows on
    the few rows of the batch's tokens."""
    from trainingjob_operator_b200.models.gpt2 import GPT2Reference
    from trainingjob_operator_b200.ops.selfcheck import _check

    env = {"AITJ_ATTN": "wgmma", "AITJ_ATTN_BWD": "wgmma"} if variant == "wgmma-attention" else None
    B, T = 2, 256
    cfg, eng = _gpu_engine(C, B=B, T=T, doc_mask=variant == "doc-mask", env=env, vocab=1000)
    assert eng.ln_impl == "wide"
    if env:
        assert eng.attn_impl == "wgmma" and eng.attn_bwd_impl == "wgmma"
    ref = GPT2Reference(cfg, eng.params).cuda()
    g = torch.Generator().manual_seed(5)
    tok = torch.randint(0, cfg.vocab_size, (B, T), generator=g).cuda()
    tgt = torch.roll(tok, -1, dims=1)
    eng.tok.copy_(tok.view(-1))
    eng.tgt.copy_(tgt.view(-1))
    doc = None
    if variant == "doc-mask":
        doc = torch.zeros(B, T, dtype=torch.int32)
        doc[:, 100:] = 100                                  # two documents per row
        doc[1, 180:] = 180
        doc = doc.cuda()
        eng.doc_start.copy_(doc.view(-1))
    eng.params.g32.zero_()
    eng.forward()
    eng.backward()
    torch.cuda.synchronize()
    rl = ref(tok, tgt, doc)
    rl.backward()
    ok = _check("loss", eng.loss, rl.detach().reshape(1), 5e-3)
    for name in ("wte", "wpe", "h0.qkv_w", "h0.qkv_b", "h0.proj_w", "h0.fc_w", "h0.fc_b", "h0.fc2_w", "h1.ln1_w",
                 "h1.ln2_b", "h1.fc2_w", "lnf_w", "lnf_b"):
        ok &= _check(f"grad {name}", eng.params.grad(name), ref.p(name).grad, 4e-2, rtol=1e-1, atol_scale=2.5e-1)
    assert ok


@pytest.mark.gpu
def test_eval_forward_at_xl_width_agrees_with_forward():
    cfg, eng = _gpu_engine(1600, B=4, T=256)
    g = torch.Generator().manual_seed(5)
    tok = torch.randint(0, cfg.vocab_size, (4 * 256,), generator=g)
    eng.tok.copy_(tok)
    eng.tgt.copy_(torch.roll(tok, -1))
    loss = float(eng.forward())
    eng.eval_acc.zero_()
    acc = eng.eval_forward()
    torch.cuda.synchronize()
    assert float(acc[1]) == 4 * 256
    assert abs(float(acc[0] / acc[1]) - loss) < 2e-3 * loss, (float(acc[0] / acc[1]), loss)


@pytest.mark.gpu
def test_greedy_decoding_at_xl_width_follows_the_reference_argmax():
    from trainingjob_operator_b200.models.generate import GPT2Generator
    from trainingjob_operator_b200.models.gpt2 import GPT2Reference

    cfg, eng = _gpu_engine(1600, B=1, T=128, seed=11)
    with torch.no_grad():                               # sharper logits than at initialisation: clear margins
        eng.params.w32("wte").mul_(25.0)
        eng.params.refresh_compute_copy()
    ref = GPT2Reference(cfg, eng.params).cuda()
    prompt, n = [5, 17, 400], 12
    out = GPT2Generator(eng, 2, len(prompt) + n).generate(prompt, n, temperature=0.0)
    seq = torch.tensor([prompt, prompt], device="cuda")
    seen = {}
    ce = torch.nn.functional.cross_entropy

    def grab(logits, target, *a, **k):
        seen["z"] = logits
        return ce(logits, target, *a, **k)

    torch.nn.functional.cross_entropy = grab
    try:
        with torch.no_grad():
            for _ in range(n):
                ref(seq, torch.zeros_like(seq))
                z = seen["z"].view(2, seq.shape[1], -1)[:, -1]
                top2 = torch.topk(z, 2, dim=-1).values
                assert float((top2[:, 0] - top2[:, 1]).min()) > 0.02 * float(z.abs().max()), "margins too small"
                seq = torch.cat([seq, torch.argmax(z, -1, keepdim=True)], 1)
    finally:
        torch.nn.functional.cross_entropy = ce
    assert torch.equal(out.cpu(), seq.cpu()), (out.tolist(), seq.tolist())


@pytest.mark.gpu
@pytest.mark.parametrize("name,batch", [("gpt2", 8), ("gpt2-medium", 8), ("gpt2-large", 4), ("gpt2-xl", 4)])
def test_every_size_trains_at_full_depth(name, batch):
    from trainingjob_operator_b200.models.gpt2 import GPT2Engine

    cfg = gpt2_config(name)
    eng = GPT2Engine(cfg, batch, 1024, "cuda", seed=0)
    g = torch.Generator().manual_seed(0)
    tok = torch.randint(0, cfg.vocab_size, (batch * 1024,), generator=g)
    eng.tok.copy_(tok)
    eng.tgt.copy_(torch.roll(tok, -1))
    losses = []
    for step in range(1, 6):
        eng.forward()
        eng.backward()
        eng.optimizer_step(lr=3e-4, step=step)
        losses.append(float(eng.loss))
    print(name, losses)
    assert all(math.isfinite(x) for x in losses) and losses[-1] < losses[0] - 0.1, losses
    del eng
    torch.cuda.empty_cache()
