"""The wgmma GEMM's epilogue variants, checked without a GPU.

The epilogue is a template parameter of the kernel (``kEpi``, the EPI_* bits), so each kernel contains only the paths
its variant uses.  With the variant tested at run time instead, every kernel carried every path -- about 19,900 SASS
instructions for a 256-wide tile -- and the consumer warps fetched that code again for every tile, which cost a K = 768
GEMM more than half its time.  These tests compile ``gemm_wgmma.cu`` for sm_90a and bound what each instantiation
contains, and check that every GEMM the engines issue has a kernel and that any other combination is refused by name.
"""
import re

import pytest
import torch

import kernel_emulation as ke
from test_gemm_sass import gemm_sass  # noqa: F401  (module fixture: name -> SASS lines of every GEMM instantiation)
from trainingjob_operator_b200.ops import functional as F

# A plain-store or bias epilogue compiles to under 1,100 instructions and the largest variant without GELU (the
# owner-sharded weight gradient, which looks up the owner of every element) to about 4,700; GELU and dGELU add one
# MUFU.TANH per output element, and the dGELU + column-sum variant is about 5,900.  The budgets leave room for compiler
# drift and stay far below the ~19,900 of an epilogue that carries every path.
BUDGET = 5000
BUDGET_GELU = 6500


def _opcode(line):
    ins = line.split("*/", 1)[1].strip()
    ins = re.sub(r"^@!?U?P\w+\s+", "", ins)
    return ins.split()[0] if ins else ""


@pytest.fixture(scope="module")
def variants(gemm_sass):  # noqa: F811
    """(block_n, a_mn, b_mn, cluster size, epilogue bits) -> opcodes of that instantiation."""
    out = {}
    for name, lines in gemm_sass.items():
        keys = ke.gemm_kernel_keys([name])
        assert keys, f"{name}: the GEMM kernel has no epilogue template parameter"
        out[keys.pop()] = [_opcode(s) for s in lines]
    return out


def test_the_emulated_kernel_table_is_the_compiled_one(variants):
    """The GEMM stand-in refuses (-7) what the built library has no kernel for; it reads the instantiations from the
    library's registered kernel names, which must be the ones compiled here."""
    assert ke.compiled_gemm_kernels() == set(variants)


def _gelu(epi):
    return bool(epi & (F.EPI_GELU | F.EPI_DGELU))


def test_every_instantiation_fits_its_instruction_budget(variants):
    over = {k: len(ops) for k, ops in variants.items() if len(ops) > (BUDGET_GELU if _gelu(k[4]) else BUDGET)}
    assert not over, f"instantiations over budget ({BUDGET} / {BUDGET_GELU} with GELU): {over}"


def test_no_tanh_without_gelu(variants):
    bad = {k: ops.count("MUFU.TANH") for k, ops in variants.items() if not _gelu(k[4]) and "MUFU.TANH" in ops}
    assert not bad, f"MUFU.TANH in variants without GELU or dGELU: {bad}"


def test_no_reduction_in_bf16_outputs_without_column_sums(variants):
    plain = [k for k in variants if not k[4] & (F.EPI_OUT_F32 | F.EPI_ACCUM | F.EPI_COLSUM)]
    assert plain
    bad = {k: sorted({o for o in variants[k] if re.match(r"(RED|ATOM)", o)}) for k in plain}
    bad = {k: v for k, v in bad.items() if v}
    assert not bad, f"global reductions or atomics in bf16 variants without column sums: {bad}"


def _compiled_pairs(variants):
    """(a_mn, b_mn, epilogue) pairs compiled for every tile configuration (128 / 256 wide, clusters of 2 and 4)."""
    tiles = {(128, 1), (256, 1), (256, 2), (256, 4)}
    got = {}
    for bn, amn, bmn, cm, epi in variants:
        got.setdefault((amn, bmn, epi), set()).add((bn, cm))
    return {k for k, v in got.items() if v == tiles}


def _record(monkeypatch):
    calls = set()

    def gemm(a, b, out, *, a_mn=False, b_mn=False, **kw):
        epi = F.gemm_epilogue(out, **{k: v for k, v in kw.items() if k not in ("split_k", "block_n", "max_ctas")})
        calls.add((bool(a_mn), bool(b_mn), epi))
        return ke.gemm(a, b, out, a_mn=a_mn, b_mn=b_mn, **kw)

    monkeypatch.setattr(F, "gemm", gemm)
    return calls


def _gpt2():
    from trainingjob_operator_b200.models.gpt2 import GPT2Config, GPT2Engine

    cfg = GPT2Config(vocab_size=1000, n_layer=2, n_head=4, n_embd=256, block_size=128, name="t")
    return GPT2Engine(cfg, 2, 128, "cpu", seed=3, gemm_backend="wgmma")


@pytest.mark.parametrize("mode", ["gpt2", "gpt2-no-pair", "gpt2-owner-sharded", "bert"])
def test_every_gemm_the_engines_issue_has_a_kernel(monkeypatch, variants, mode):
    ke.install(monkeypatch)
    calls = _record(monkeypatch)
    if mode == "gpt2-no-pair":
        monkeypatch.setenv("AITJ_GEMM_PAIR", "0")
    if mode == "bert":
        from trainingjob_operator_b200.models.bert import BertConfig, BertEngine

        eng = BertEngine(BertConfig.tiny(), 2, 128, "cpu", seed=3)
    else:
        eng = _gpt2()
    if mode == "gpt2-owner-sharded":
        fw = ke.FakeWorld(2)
        fw.attach(eng.params)
        fw.attach(_gpt2().params)
    eng.forward()
    eng.backward()
    expected = {(False, False, F.EPI_BIAS), (False, True, F.EPI_DGELU | F.EPI_COLSUM)}
    if mode == "gpt2-no-pair":
        expected = {(False, False, F.EPI_BIAS), (False, True, F.EPI_DGELU)}
    if mode == "gpt2-owner-sharded":
        expected.add((True, True, F.EPI_ACCUM | F.EPI_PEER))
    assert expected <= calls, calls           # the recorder sees the fused epilogues
    missing = {(a, b, F.epilogue_name(e)) for a, b, e in calls - _compiled_pairs(variants)}
    assert not missing, f"GEMMs without a compiled kernel: {missing}"


def test_a_gemm_without_a_kernel_is_refused_by_name(monkeypatch):
    """The library answers an unlisted (layout, epilogue) pair with its own error code before it touches the device;
    ``functional.gemm`` turns that into an exception naming the pair."""
    monkeypatch.setattr(F, "_stream", lambda: 0)
    a = torch.zeros(256, 128, dtype=torch.bfloat16)
    b = torch.zeros(256, 128, dtype=torch.bfloat16)
    out = torch.zeros(128, 128, dtype=torch.bfloat16)
    bias = torch.zeros(128, dtype=torch.bfloat16)
    with pytest.raises(F.lib.KernelError, match=r"a_mn=1 b_mn=1 with epilogue BIAS\b") as e:
        F.gemm(a, b, out, a_mn=True, b_mn=True, bias=bias)
    assert e.value.code == F.GEMM_NO_KERNEL
    res = torch.zeros(128, 128, dtype=torch.bfloat16)
    cs = torch.zeros(128, dtype=torch.float32)
    with pytest.raises(F.lib.KernelError, match=r"a_mn=0 b_mn=1 with epilogue RESIDUAL\|COLSUM"):
        F.gemm(a.t().contiguous(), b, out, b_mn=True, residual=res, colsum=cs)
