"""Device-timed microbenchmarks of the hand-written kernels vs. the library path (cuBLAS).

CUDA events on the launching stream, >=3 warm-ups, L2 flushed (write of a 256 MiB buffer)
between timed iterations.  Writes gpurun_out/kernel_bench.json and prints a table.
"""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from trainingjob_operator_b200.ops import functional as F  # noqa: E402

PEAKS = {}
try:
    PEAKS = json.load(open(os.path.join(os.path.dirname(__file__), "..", "MEASURED_PEAKS.json")))
except Exception:
    pass
# shares of a peak are only reported against peaks measured on the same card (MEASURED_PEAKS.json); null otherwise
PEAK_TF = PEAKS.get("bf16_tflops")
PEAK_BW = PEAKS.get("hbm_gbs")


def frac(rate, peak):
    return rate / peak if peak else None

_flush = None


def flush_l2():
    global _flush
    if _flush is None:
        _flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")
    _flush.fill_(1)


def timeit(fn, iters=10, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        flush_l2()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[len(ts) // 2], ts[0]


def main():
    rows = []
    B, T, C = 16, 1024, 768
    M = B * T
    shapes = [
        ("qkv fwd", M, 3 * C, C, False, False),
        ("attn proj fwd", M, C, C, False, False),
        ("fc fwd", M, 4 * C, C, False, False),
        ("fc2 fwd", M, C, 4 * C, False, False),
        ("lm_head fwd", M, 50304, C, False, False),
        ("fc dgrad", M, C, 4 * C, False, True),
        ("fc2 dgrad", M, 4 * C, C, False, True),
        ("lm_head dgrad", M, C, 50304, False, True),
        ("square 8192", 8192, 8192, 8192, False, False),
        ("square 4096", 4096, 4096, 4096, False, False),
    ]
    mem_only = "--mem-only" in sys.argv
    for name, m, n, k, a_mn, b_mn in ([] if mem_only else shapes):
        a = torch.randn(m, k, device="cuda").bfloat16()
        b = (torch.randn(k, n, device="cuda") if b_mn else torch.randn(n, k, device="cuda")).bfloat16()
        out = torch.empty(m, n, device="cuda", dtype=torch.bfloat16)
        flops = 2.0 * m * n * k
        for bn in (1024, 512, 256):
            med, best = timeit(lambda: F.gemm(a, b, out, a_mn=a_mn, b_mn=b_mn, block_n=bn))
            rows.append({"kernel": f"wgmma {name} bn={bn}", "M": m, "N": n, "K": k, "ms_med": med, "ms_best": best,
                         "tflops": flops / med / 1e9, "frac_of_measured_peak": frac(flops / med / 1e9, PEAK_TF)})
        bt = b if b_mn else b.t()
        med, best = timeit(lambda: torch.matmul(a, bt, out=out))
        rows.append({"kernel": f"cublas  {name}", "M": m, "N": n, "K": k, "ms_med": med, "ms_best": best,
                     "tflops": flops / med / 1e9, "frac_of_measured_peak": frac(flops / med / 1e9, PEAK_TF)})
    # wgrad (split-K, fp32 red.add)
    for name, nout, kin in ([] if mem_only else [("qkv wgrad", 3 * C, C), ("fc wgrad", 4 * C, C), ("fc2 wgrad", C, 4 * C),
                                                 ("proj wgrad", C, C), ("lm_head wgrad", 50304, C)]):
        dy = torch.randn(M, nout, device="cuda").bfloat16()
        x = torch.randn(M, kin, device="cuda").bfloat16()
        dw = torch.zeros(nout, kin, device="cuda")
        sk = F.auto_split_k(nout, kin, M)
        flops = 2.0 * M * nout * kin
        for bn, tag in ((1024, "quad"), (512, "2cta"), (0, "1cta")):
            skk = F.auto_split_k(nout, kin, M, 256) * (2 if bn >= 512 else 1)
            med, best = timeit(lambda: F.gemm(dy, x, dw, a_mn=True, b_mn=True, accumulate=True, split_k=skk, block_n=bn))
            rows.append({"kernel": f"wgmma {name} {tag} sk={skk}", "M": nout, "N": kin, "K": M, "ms_med": med,
                         "ms_best": best, "tflops": flops / med / 1e9,
                         "frac_of_measured_peak": frac(flops / med / 1e9, PEAK_TF)})
        med, best = timeit(lambda: F.gemm(dy, x, dw, a_mn=True, b_mn=True, accumulate=True, split_k=sk))
        rows.append({"kernel": f"wgmma {name} sk={sk}", "M": nout, "N": kin, "K": M, "ms_med": med, "ms_best": best,
                     "tflops": flops / med / 1e9, "frac_of_measured_peak": frac(flops / med / 1e9, PEAK_TF)})
        dwb = torch.empty(nout, kin, device="cuda", dtype=torch.bfloat16)
        med, best = timeit(lambda: torch.matmul(dy.t(), x, out=dwb))
        rows.append({"kernel": f"cublas  {name}", "M": nout, "N": kin, "K": M, "ms_med": med, "ms_best": best,
                     "tflops": flops / med / 1e9, "frac_of_measured_peak": frac(flops / med / 1e9, PEAK_TF)})

    # memory-bound kernels
    x = torch.randn(M, C, device="cuda").bfloat16()
    g = torch.ones(C, device="cuda").bfloat16()
    bta = torch.zeros(C, device="cuda").bfloat16()
    y = torch.empty_like(x)
    mean = torch.empty(M, device="cuda")
    rstd = torch.empty(M, device="cuda")
    med, best = timeit(lambda: F.layernorm_fwd(x, g, bta, y, mean, rstd))
    byts = 2 * M * C * 2
    rows.append({"kernel": "layernorm fwd", "ms_med": med, "ms_best": best, "gbs": byts / med / 1e6,
                 "frac_of_measured_peak": frac(byts / med / 1e6, PEAK_BW)})
    dx = torch.empty_like(x)
    dg = torch.zeros(C, device="cuda")
    dbt = torch.zeros(C, device="cuda")
    med, best = timeit(lambda: F.layernorm_bwd(y, x, g, mean, rstd, dx, dg, dbt, dres=x))
    byts = 4 * M * C * 2
    rows.append({"kernel": "layernorm bwd(+dres)", "ms_med": med, "ms_best": best, "gbs": byts / med / 1e6,
                 "frac_of_measured_peak": frac(byts / med / 1e6, PEAK_BW)})
    Vp = 50304
    logits = torch.randn(M, Vp, device="cuda").bfloat16()
    tgt = torch.randint(0, 50257, (M,), device="cuda")
    loss = torch.empty(M, device="cuda")
    med, best = timeit(lambda: F.softmax_xent(logits, tgt, loss, 50257, 1.0 / M), iters=5)
    byts = 2 * M * Vp * 2
    rows.append({"kernel": "softmax_xent fwd+bwd", "ms_med": med, "ms_best": best, "gbs": byts / med / 1e6,
                 "frac_of_measured_peak": frac(byts / med / 1e6, PEAK_BW)})
    del logits
    n = 124_475_904 // 256 * 256
    p = torch.randn(n, device="cuda")
    gr = torch.randn(n, device="cuda")
    m1 = torch.zeros(n, device="cuda")
    v1 = torch.zeros(n, device="cuda")
    p16 = torch.empty(n, device="cuda", dtype=torch.bfloat16)
    mask = torch.ones(n // 256, dtype=torch.uint8, device="cuda")
    ss = torch.zeros(1, device="cuda")
    med, best = timeit(lambda: F.adamw(p, gr, m1, v1, p16, mask, lr=1e-4, step=3, sumsq_buf=ss, max_norm=1.0))
    byts = n * (16 + 16 + 2)
    rows.append({"kernel": "adamw flat (fp32 p,g,m,v + bf16 copy + zero g)", "ms_med": med, "ms_best": best,
                 "gbs": byts / med / 1e6, "frac_of_measured_peak": frac(byts / med / 1e6, PEAK_BW)})
    med, best = timeit(lambda: F.sumsq(gr, ss))
    rows.append({"kernel": "sumsq", "ms_med": med, "ms_best": best, "gbs": n * 4 / med / 1e6,
                 "frac_of_measured_peak": n * 4 / med / 1e6 / PEAK_BW})

    os.makedirs("gpurun_out", exist_ok=True)
    json.dump({"peaks": {"bf16_tflops": PEAK_TF, "hbm_gbs": PEAK_BW}, "rows": rows},
              open("gpurun_out/kernel_bench.json", "w"), indent=1)
    for r in rows:
        perf = f"{r['tflops']:8.1f} TF" if "tflops" in r else f"{r['gbs']:8.1f} GB/s"
        print(f"{r['kernel']:<52s} {r['ms_med']:8.3f} ms  {perf}  {100 * r['frac_of_measured_peak']:5.1f}% of measured")


if __name__ == "__main__":
    main()
