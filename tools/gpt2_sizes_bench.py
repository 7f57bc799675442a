"""GPT-2 small, medium, large and XL on one H100: step time, throughput and peak memory per size, and the LayerNorm
kernels at each width they serve.

    python tools/gpt2_sizes_bench.py --out DIR [--steps 10] [--iters 200] [--rounds 3]

Prints the card and its power limit and writes ``DIR/gpt2_sizes.json``.  All times are CUDA-event times after warm-up.

* Per size, at one GPU, T = 1024 and the per-GPU batch the README recommends: the graph-replayed training step
  (``EngineTrainer``, as a worker runs it) over ``--steps`` steps; tokens/s; model TFLOP/s from ``flops_per_token`` and
  its share of the 989 TFLOP/s dense BF16 data-sheet figure (a whole-program share, not a kernel's); and the peak
  ``torch.cuda.max_memory_allocated`` of the steps, without and with the device snapshot ``AsyncCheckpointer.save``
  allocates (one buffer per state tensor, filled by a device copy; the snapshot is not written to disk here).  XL is
  also tried at batch 16, where it may not fit: that is recorded, not raised.
* LayerNorm forward and backward (with dres and dxsum, as the engine calls it) at M = 16384 (B16 x T1024) for each width
  and kernel pair the engines use, and both pairs at 1024: the arms alternate ``--rounds`` times, ``--iters`` launches
  each, and the bytes each kernel must move are computed from the shapes below.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PEAK_TFLOPS = 989.0            # H100 SXM data sheet, dense BF16
SIZES = [("gpt2", 16), ("gpt2-medium", 16), ("gpt2-large", 16), ("gpt2-xl", 8), ("gpt2-xl", 16)]
LN_ARMS = [(768, "fused"), (1024, "fused"), (1024, "wide"), (1280, "wide"), (1600, "wide")]


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = [x.strip() for x in r.stdout.splitlines()[0].split(",")]
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def bench_size(name, B, steps):
    import torch

    from trainingjob_operator_b200.models.gpt2 import GPT2Engine, flops_per_token, gpt2_config
    from trainingjob_operator_b200.runtime.trainer import EngineTrainer, SyntheticTokens

    cfg, T = gpt2_config(name), 1024
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    rec = {"model": name, "batch": B, "seq": T}
    try:
        eng = GPT2Engine(cfg, B, T, "cuda", seed=0)
        data = SyntheticTokens(cfg.vocab_size, B, T, n_batches=4, seed=1)
        tr = EngineTrainer(eng, lr=3e-4, use_graph=True)
        for _ in range(3):
            tr.step(*data.next())
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            tr.step(*data.next(), read_loss=False)
        e1.record()
        e1.synchronize()
        ms = e0.elapsed_time(e1) / steps
        loss = float(eng.loss)
        peak = torch.cuda.max_memory_allocated()
        tflops = flops_per_token(cfg, T) * B * T / (ms * 1e-3) / 1e12
        rec.update(params=eng.num_parameters(), cuda_graph=tr.graph is not None, ms_per_step=round(ms, 3),
                   tokens_per_s=round(B * T / (ms * 1e-3)), model_tflops=round(tflops, 1),
                   whole_program_share_of_989_tflops=round(tflops / PEAK_TFLOPS, 4), loss_after=round(loss, 4),
                   peak_gb=round(peak / 1e9, 2), fits=True)
        try:
            snap = [torch.empty_like(t) for t in tr.state_tensors()]
            for d, s in zip(snap, tr.state_tensors()):
                d.copy_(s)
            tr.step(*data.next())
            torch.cuda.synchronize()
            rec.update(snapshot_gb=round(sum(t.numel() * t.element_size() for t in snap) / 1e9, 2),
                       peak_with_snapshot_gb=round(torch.cuda.max_memory_allocated() / 1e9, 2), fits_with_snapshot=True)
            del snap
        except torch.OutOfMemoryError:
            rec.update(fits_with_snapshot=False)
        del tr, eng
    except torch.OutOfMemoryError:
        rec.update(fits=False, fits_with_snapshot=False)
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    print(json.dumps(rec), flush=True)
    return rec


def _time(fn, iters):
    import torch

    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / iters


def bench_layernorm(iters, rounds, M=16384):
    import torch

    from trainingjob_operator_b200.ops import functional as F

    g = torch.Generator(device="cuda").manual_seed(0)
    arms = {}
    for C, impl in LN_ARMS:
        x, dy, dres = (torch.randn(M, C, device="cuda", generator=g).bfloat16() for _ in range(3))
        gamma, beta = torch.randn(C, device="cuda", generator=g).bfloat16(), torch.zeros(C, device="cuda").bfloat16()
        y, dx = torch.empty_like(x), torch.empty_like(x)
        mean, rstd = torch.empty(M, device="cuda"), torch.empty(M, device="cuda")
        grads = torch.zeros(3, C, device="cuda")
        fwd, bwd = (F.layernorm_fwd, F.layernorm_bwd) if impl == "fused" else (F.layernorm_wide_fwd, F.layernorm_wide_bwd)
        arms[(C, impl)] = {
            "fwd": (lambda fwd=fwd, x=x, gamma=gamma, beta=beta, y=y, mean=mean, rstd=rstd:
                    fwd(x, gamma, beta, y, mean, rstd)),
            "bwd": (lambda bwd=bwd, dy=dy, x=x, gamma=gamma, mean=mean, rstd=rstd, dx=dx, grads=grads, dres=dres:
                    bwd(dy, x, gamma, mean, rstd, dx, grads[0], grads[1], dres=dres, dxsum=grads[2])),
            # HBM bytes the kernel cannot avoid: forward reads x, gamma, beta and writes y, mean, rstd; backward reads
            # dy, x, dres, gamma, mean, rstd and writes dx (the C-wide parameter-gradient adds are left out)
            "bytes": {"fwd": 2 * M * C * 2 + 2 * C * 2 + 2 * M * 4, "bwd": 4 * M * C * 2 + C * 2 + 2 * M * 4},
        }
        for k in ("fwd", "bwd"):
            arms[(C, impl)][k]()
    torch.cuda.synchronize()
    times = {key: {"fwd": [], "bwd": []} for key in arms}
    for _ in range(rounds):
        for key, a in arms.items():
            for k in ("fwd", "bwd"):
                times[key][k].append(_time(a[k], iters))
    out = []
    for (C, impl), a in arms.items():
        rec = {"C": C, "kernels": impl, "M": M}
        for k in ("fwd", "bwd"):
            best = min(times[(C, impl)][k])
            rec[f"{k}_us"] = round(best * 1e3, 2)
            rec[f"{k}_us_all"] = [round(t * 1e3, 2) for t in times[(C, impl)][k]]
            rec[f"{k}_gbs"] = round(a["bytes"][k] / (best * 1e-3) / 1e9, 1)
        out.append(rec)
        print(json.dumps(rec), flush=True)
    base = next(r for r in out if r["C"] == 768)
    for r in out:
        r["fwd_rate_vs_fused_768"] = round(r["fwd_gbs"] / base["fwd_gbs"], 3)
        r["bwd_rate_vs_fused_768"] = round(r["bwd_gbs"] / base["bwd_gbs"], 3)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("gpt2_sizes_bench needs a GPU")
    res = {"card": card()}
    print(json.dumps(res["card"]), flush=True)
    res["layernorm"] = bench_layernorm(args.iters, args.rounds)
    res["sizes"] = [bench_size(name, B, args.steps) for name, B in SIZES]
    res["card_after"] = card()
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "gpt2_sizes.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
