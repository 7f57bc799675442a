"""The wgmma GEMM's bf16 epilogues leave through shared memory and TMA, checked without a GPU.

A bf16 epilogue that stores from the accumulator registers issues one 32-bit store per fragment pair: each warp store
covers 8 rows x 16 bytes, eight partial writes to eight lines, and every SM issues them at the same moment.  With
those stores behind a condition that is never true, GPT-2's lm_head forward took 1.55 instead of 2.76 ms on an H100.
The epilogue now writes swizzled 64 x 64 boxes into shared memory and stores them with TMA, and the residual and saved
pre-activation it reads arrive the same way.
"""
import pytest
import torch

from test_gemm_sass import gemm_sass  # noqa: F401  (module fixture: name -> SASS lines of every GEMM instantiation)
from test_gemm_epilogue_variants import variants  # noqa: F401  (module fixture: instantiation -> opcodes)
from trainingjob_operator_b200.ops import functional as F


def _bf16(epi):
    return not epi & (F.EPI_OUT_F32 | F.EPI_ACCUM)


def test_bf16_outputs_leave_by_tma_store(variants):  # noqa: F811
    bf16 = [k for k in variants if _bf16(k[4])]
    assert bf16
    bad = {k: sorted({o for o in variants[k] if o.startswith("STG")}) for k in bf16}
    bad = {k: v for k, v in bad.items() if v}
    assert not bad, f"global stores in bf16 epilogues: {bad}"
    missing = [k for k in bf16 if not any(o.startswith("UTMASTG") for o in variants[k])]
    assert not missing, f"bf16 epilogues without a TMA store: {missing}"


def test_residual_and_gelu_inputs_arrive_by_tma(variants):  # noqa: F811
    """A RESIDUAL or DGELU instantiation loads no more from global memory than the same kernel without those bits: its
    only LDG are the bias loads."""
    reads = [k for k in variants if _bf16(k[4]) and k[4] & (F.EPI_RESIDUAL | F.EPI_DGELU)]
    assert reads
    count = {k: sum(o.startswith("LDG") for o in ops) for k, ops in variants.items()}
    bad = {}
    for k in reads:
        base = k[:4] + (k[4] & F.EPI_BIAS,)
        assert base in variants, f"{k}: no instantiation {base} to compare with"
        if count[k] > count[base]:
            bad[k] = (count[k], count[base])
    assert not bad, f"LDG in RESIDUAL / DGELU epilogues beyond the variant without them (got, base): {bad}"
    missing = [k for k in reads if not any(o.startswith("UTMALDG") for o in variants[k])]
    assert not missing


@pytest.mark.parametrize("what", ["residual", "aux"])
def test_a_misaligned_epilogue_input_is_refused(monkeypatch, what):
    """TMA needs 16-byte aligned tensors: the library refuses a residual or aux tensor that is not, with its error code,
    before it touches the device."""
    monkeypatch.setattr(F, "_stream", lambda: 0)
    M, N, K = 128, 128, 128
    a = torch.zeros(M, K, dtype=torch.bfloat16)
    b = torch.zeros(N, K, dtype=torch.bfloat16)
    out = torch.zeros(M, N, dtype=torch.bfloat16)
    shifted = torch.zeros(M * N + 8, dtype=torch.bfloat16)[1:M * N + 1].view(M, N)   # 2 bytes past a 16-byte boundary
    assert shifted.data_ptr() % 16 and shifted.stride(0) == out.stride(0)
    kw = {"bias": torch.zeros(N, dtype=torch.bfloat16), "residual": shifted} if what == "residual" else \
         {"dgelu": True, "aux": shifted}
    with pytest.raises(F.lib.KernelError) as e:
        F.gemm(a, b, out, **kw)
    assert e.value.code == F.GEMM_MISALIGNED
