"""Micro-batch accumulation on one H100: device time of an optimizer step that accumulates k micro-batches against the
plain single-micro-batch step.

    python tools/accumulation_bench.py --out DIR [--steps 10] [--rounds 3] [--models gpt2,bert]

Prints the card and its power limit and writes ``DIR/accumulation_bench.json``.  GPT-2 small at B16 T1024 and BERT-base
at B16 T512, one GPU, CUDA graphs, synthetic inputs copied from pinned host memory before every micro-batch.  The arms
are the plain step (global batch 16) and accumulated steps of global batch 64 and 256 (k = 4, 16 micro-batches); for
each model the arms run in turn ``--rounds`` times on one engine, ``--steps`` timed steps each after the arm's graph
capture and one untimed step.  Times are CUDA-event times over the timed steps (each step reads its loss back, as the
worker's do); reported per optimizer step, per micro-batch, and per micro-batch relative to the plain step.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = [x.strip() for x in r.stdout.splitlines()[0].split(",")]
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def bench_model(model: str, globals_, steps: int, rounds: int):
    import torch

    from trainingjob_operator_b200.runtime.trainer import EngineTrainer, SyntheticTokens

    B = 16
    if model == "gpt2":
        from trainingjob_operator_b200.models.gpt2 import GPT2Config, GPT2Engine

        cfg, T = GPT2Config.small(), 1024
        eng = GPT2Engine(cfg, B, T, "cuda", seed=0)
        data = SyntheticTokens(cfg.vocab_size, B, T, n_batches=4, seed=1)
    else:
        from trainingjob_operator_b200.models.bert import BertConfig, BertEngine, SyntheticMLM

        cfg, T = BertConfig.base(), 512
        eng = BertEngine(cfg, B, T, "cuda", seed=0)
        data = SyntheticMLM(cfg.vocab_size, B, T, n_batches=4, seed=1)
    trainers = {}
    for G in globals_:
        tr = EngineTrainer(eng, lr=3e-4, use_graph=True, global_batch=G)
        trainers[G] = tr
    times = {G: [] for G in globals_}

    def one_step(tr):
        if tr.plan.accumulates:
            return tr.accumulate(data.next() for _ in range(tr.plan.n))
        return tr.step(*data.next())

    for tr in trainers.values():             # capture + one untimed step per arm
        one_step(tr)
        one_step(tr)
        assert tr.graph is not None, tr.graph_error
    for _ in range(rounds):
        for G, tr in trainers.items():
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(steps):
                loss = one_step(tr)
            e1.record()
            torch.cuda.synchronize()
            assert loss == loss
            times[G].append(e0.elapsed_time(e1) / steps)
    plain = min(times[globals_[0]])
    arms = []
    for G, tr in trainers.items():
        ms = min(times[G])
        k = tr.plan.k
        arms.append({"global_batch": G, "micro_batches": k, "ms_per_step": round(ms, 3),
                     "ms_per_micro_batch": round(ms / k, 3), "per_micro_batch_vs_plain": round(ms / k / plain, 4),
                     "samples_per_sec": round(G / ms * 1e3, 1), "ms_per_step_rounds": [round(t, 3) for t in times[G]],
                     "launches_per_step": tr.launches_per_step})
    return {"model": model, "shape": f"B{B} T{T}", "arms": arms}


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--models", default="gpt2,bert")
    args = ap.parse_args()
    import torch

    c = card()
    print(json.dumps(c), flush=True)
    out = {"card": c, "steps": args.steps, "rounds": args.rounds, "gpus": 1, "results": [],
           "unmeasured": ["owner-sharded (rs) accumulation on 2 GPUs: this run had "
                          f"{torch.cuda.device_count()} GPU(s)"] if torch.cuda.device_count() < 2 else []}
    for model in args.models.split(","):
        r = bench_model(model, [16, 64, 256], args.steps, args.rounds)
        print(json.dumps(r), flush=True)
        out["results"].append(r)
        torch.cuda.empty_cache()
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "accumulation_bench.json"), "w") as f:
        json.dump(out, f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
