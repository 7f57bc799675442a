"""Decode-path timing of GPT-2 small on one GPU: ms per generated token, per-kernel time, attention bandwidth.

    python tools/generate_bench.py --out DIR

* ms per generated token at S in {1, 4, 16} sequences and contexts 64 / 512 / 1024: one generation of a one-token
  prompt and ctx - 1 new tokens, timed with CUDA events and divided by its ctx - 1 decode steps -- the mean over
  positions 0 .. ctx - 2 -- with the step replayed as a CUDA graph (the figure includes the first, eager step and the
  capture) and launched eagerly;
* each decode kernel's device time per step (torch.profiler's kernel durations) over a generation of 1024 tokens, and
  the GEMMs' share of the step's kernel time;
* ``attention_decode`` at pos = 1023: device time per call (its two kernels' durations over 200 calls) and the bytes it
  must move -- this layer's K and V cache of S x 1024 positions, the new qkv row, the output -- over that time, against
  the H100 SXM data sheet's 3.35 TB/s.

The bound of a decode step is the weights: every token reads the 124M bf16 parameters (248 MB), at least 0.074 ms at
3.35 TB/s.  The card name and its power limit are read in the same run and written with the numbers.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = (x.strip() for x in q.stdout.splitlines()[0].split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def time_generation(gen, S, ctx, use_graph):
    steps = ctx - 1
    gen.generate([50256], 8, temperature=1.0, top_k=50, seed=1, use_graph=use_graph)      # warm-up
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    gen.generate([50256], steps, temperature=1.0, top_k=50, seed=2, use_graph=use_graph)
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / steps


def kernel_times(fn) -> dict:
    """{kernel name: total device microseconds} of the kernels ``fn`` launches (torch.profiler, CUDA activity)."""
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", 0) or getattr(e, "cuda_time_total", 0)
        if us > 0 and not e.key.startswith(("Memcpy", "Memset")):
            name = e.key.split("(")[0].replace("void ", "")[:100]
            out[name] = out.get(name, 0.0) + us
    return out


def main(argv=None) -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("generate_bench needs a GPU")
    from trainingjob_operator_b200.models.generate import GPT2Generator
    from trainingjob_operator_b200.models.gpt2 import GPT2Config, GPT2Engine
    from trainingjob_operator_b200.ops import functional as F

    torch.cuda.set_device(0)
    res = {"card": card(), "model": "gpt2-small", "weights_bytes": 0, "per_token_ms": [], "kernels": {},
           "attention_decode_pos1023": []}
    cfg = GPT2Config.small()
    eng = GPT2Engine(cfg, 1, 1, "cuda", seed=0)
    res["weights_bytes"] = eng.num_parameters() * 2
    res["weights_bound_ms"] = res["weights_bytes"] / HBM_BYTES_PER_S * 1e3
    for S in (1, 4, 16):
        gens = {ctx: GPT2Generator(eng, S, ctx) for ctx in (64, 512, 1024)}
        for ctx, gen in gens.items():
            row = {"S": S, "context": ctx}
            for mode, g in (("graph", True), ("eager", False)):
                row[f"{mode}_ms"] = round(time_generation(gen, S, ctx, g), 4)
            print(json.dumps(row), flush=True)
            res["per_token_ms"].append(row)
        # kernel time per decode step over a generation of 1024 tokens (device durations of every kernel)
        gen = gens[1024]
        prof = kernel_times(lambda: gen.generate([50256], 1023, temperature=1.0, top_k=50, seed=3, use_graph=False))
        total = sum(prof.values())
        gemm = sum(us for k, us in prof.items() if "gemm" in k)
        res["kernels"][f"S={S}"] = {
            "per_step_us": {k: round(us / 1023, 2) for k, us in sorted(prof.items(), key=lambda kv: -kv[1])},
            "step_kernel_ms": round(total / 1023 / 1e3, 4), "gemm_share": round(gemm / total, 4)}
        print(json.dumps({"S": S, **res["kernels"][f"S={S}"]}), flush=True)
        del gens, gen
        # attention_decode alone at pos = 1023 (its two kernels' device durations)
        H, C, Tmax = cfg.n_head, cfg.n_embd, 1024
        cache = torch.randn(S, Tmax, 2, H, 64, device="cuda").bfloat16()
        qkv = torch.randn(S, 3 * C, device="cuda").bfloat16()
        out = torch.empty(S, C, device="cuda").bfloat16()
        part = torch.empty(F.decode_partials(S, H, Tmax), device="cuda")
        pos = torch.tensor([1023, 0], dtype=torch.int32, device="cuda")
        for _ in range(20):
            F.attention_decode(qkv, cache, pos, out, part, H)

        def calls():
            for _ in range(200):
                F.attention_decode(qkv, cache, pos, out, part, H)

        at = kernel_times(calls)
        us = sum(v for k, v in at.items() if "attention_decode" in k) / 200
        main_us = sum(v for k, v in at.items() if "attention_decode_kernel" in k) / 200
        nbytes = S * 1024 * 2 * C * 2 + S * 3 * C * 2 + S * C * 2
        row = {"S": S, "us_per_call": round(us, 2), "split_kernel_us": round(main_us, 2), "bytes": nbytes,
               "TB_per_s": round(nbytes / us / 1e6, 3), "share_of_3.35TB_per_s": round(nbytes / us / 1e6 / 3.35, 3)}
        print(json.dumps(row), flush=True)
        res["attention_decode_pos1023"].append(row)
        del cache
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "generate_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps({"card": res["card"], "weights_bound_ms": res["weights_bound_ms"]}))
    return 0


if __name__ == "__main__":
    sys.exit(main())
