"""Held-out evaluation on one H100: the cross-entropy head fused into the logits GEMM against the training head, the
evaluation forward against the training forward, and what evaluating every N steps costs a GPT-2 small run.

    python tools/eval_bench.py --out DIR [--iters 50] [--rounds 3]

Prints the card and its power limit and writes ``DIR/eval_bench.json``.  Three measurements, all CUDA-event times after
warm-up, the arms of each alternating ``--rounds`` times:

* head at M = 16384 (B16 x T1024), N = 50304 (GPT-2's padded vocabulary), K = 768: ``gemm_xent`` + ``xent_finish``
  against the bf16 logits GEMM + ``softmax_xent``, ``--iters`` launches each, with the HBM bytes and FLOPs each needs
  computed from the shapes;
* one ``GPT2Engine.eval_forward()`` against one ``forward()`` at GPT-2 small, B16 x T1024;
* the graph-replayed GPT-2 small training step, alone and with an evaluation of 20 micro-batches (llm.c's
  ``val_max_steps``) every 20 steps, as ``--eval-every 20`` runs it.  The overhead is evaluation time over training
  time (how much longer the run takes); the share is evaluation time over the whole run's time.
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


def _time(fn, iters):
    import torch

    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / iters


def bench_head(iters, rounds):
    import torch

    from trainingjob_operator_b200.ops import functional as F

    M, N, K, V = 16384, 50304, 768, 50257
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(M, K, device="cuda", generator=g).bfloat16()
    w = (torch.randn(N, K, device="cuda", generator=g) * 0.05).bfloat16()
    tgt = torch.randint(0, V, (M,), device="cuda", generator=g)
    part = torch.empty(M, F.xent_blocks(N), 2, device="cuda")
    tl = torch.empty(M, device="cuda")
    loss = torch.empty(M, device="cuda")
    acc = torch.zeros(2, device="cuda", dtype=torch.float64)
    logits = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    loss2 = torch.empty(M, device="cuda")

    def fused():
        F.gemm_xent(x, w, tgt, V, part, tl, block_n=512)
        F.xent_finish(part, tl, tgt, loss, acc)

    def unfused():
        F.gemm(x, w, logits, block_n=512)
        F.softmax_xent(logits, tgt, loss2, V, 1.0 / M)

    for fn in (fused, unfused):
        for _ in range(5):
            fn()
    torch.cuda.synchronize()
    times = {"fused": [], "unfused": []}
    for _ in range(rounds):
        times["fused"].append(_time(fused, iters))
        times["unfused"].append(_time(unfused, iters))
    acc.zero_()
    fused()
    unfused()
    torch.cuda.synchronize()
    diff = float((loss - loss2).abs().max())
    nb = F.xent_blocks(N)
    operands = (M * K + N * K) * 2
    bytes_ = {"fused": operands + M * nb * 8 * 2 + M * (4 + 8) * 2 + M * 4,     # partials out + in, target, logit, loss
              "unfused": operands + M * N * 2 * 3 + M * (8 + 4)}               # logits out, in, dlogits out
    flops = 2.0 * M * N * K
    out = {"M": M, "N": N, "K": K, "vocab": V, "iters": iters, "flops": flops,
           "max_abs_loss_diff_fused_vs_unfused": diff}
    for arm in ("fused", "unfused"):
        ms = min(times[arm])
        out[arm] = {"ms": round(ms, 4), "ms_rounds": [round(t, 4) for t in times[arm]], "hbm_bytes": bytes_[arm],
                    "tflops": round(flops / ms / 1e9, 1), "gb_per_s_of_needed_bytes": round(bytes_[arm] / ms / 1e6, 1)}
    out["speedup"] = round(out["unfused"]["ms"] / out["fused"]["ms"], 3)
    return out


def bench_forward(iters, rounds):
    import torch

    from trainingjob_operator_b200.models.gpt2 import GPT2Config, GPT2Engine

    cfg, B, T = GPT2Config.small(), 16, 1024
    eng = GPT2Engine(cfg, B, T, "cuda", seed=0)
    tok = torch.randint(0, cfg.vocab_size, (B * T,), generator=torch.Generator().manual_seed(1))
    eng.tok.copy_(tok)
    eng.tgt.copy_(torch.roll(tok, -1))

    def ev():
        eng.eval_forward()

    for fn in (eng.forward, ev):
        for _ in range(3):
            fn()
    times = {"forward": [], "eval_forward": []}
    for _ in range(rounds):
        times["forward"].append(_time(eng.forward, iters))
        times["eval_forward"].append(_time(ev, iters))
    eng.eval_acc.zero_()
    eng.eval_forward()
    eng.forward()
    torch.cuda.synchronize()
    ev_loss = float(eng.eval_acc[0] / eng.eval_acc[1])
    out = {"model": "gpt2-small", "shape": "B16 T1024", "iters": iters,
           "loss_forward": float(eng.loss), "loss_eval_forward": ev_loss}
    for arm in times:
        out[arm] = {"ms": round(min(times[arm]), 3), "ms_rounds": [round(t, 3) for t in times[arm]]}
    del eng
    torch.cuda.empty_cache()
    return out


def bench_step(rounds, steps=40, eval_every=20, eval_micro=20):
    import torch

    from trainingjob_operator_b200.models.gpt2 import GPT2Config, GPT2Engine
    from trainingjob_operator_b200.runtime.trainer import EngineTrainer, SyntheticTokens

    cfg, B, T = GPT2Config.small(), 16, 1024
    eng = GPT2Engine(cfg, B, T, "cuda", seed=0)
    data = SyntheticTokens(cfg.vocab_size, B, T, n_batches=4, seed=1)
    held = SyntheticTokens(cfg.vocab_size, B, T, n_batches=4, seed=2)
    tr = EngineTrainer(eng, lr=3e-4, use_graph=True)
    for _ in range(3):
        tr.step(*data.next())
    tr.evaluate(held.next() for _ in range(eval_micro))

    def run(with_eval):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for s in range(1, steps + 1):
            tr.step(*data.next())
            if with_eval and s % eval_every == 0:
                tr.evaluate(held.next() for _ in range(eval_micro))
        e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1)

    def one_eval():
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        tr.evaluate(held.next() for _ in range(eval_micro))
        e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1)

    plain, with_eval, evals = [], [], []
    for _ in range(rounds):
        plain.append(run(False))
        with_eval.append(run(True))
        evals.append(one_eval())
    step_ms = min(plain) / steps
    eval_ms = min(evals)
    return {"model": "gpt2-small", "shape": "B16 T1024", "steps": steps, "eval_every": eval_every,
            "eval_micro_batches": eval_micro, "eval_samples": eval_micro * B,
            "ms_per_step": round(step_ms, 3), "ms_per_evaluation": round(eval_ms, 2),
            "ms_per_eval_micro_batch": round(eval_ms / eval_micro, 3),
            "run_ms_without_eval": [round(t, 1) for t in plain], "run_ms_with_eval": [round(t, 1) for t in with_eval],
            # overhead: evaluation time over training time (what evaluating adds to a run); share: evaluation time over
            # the whole run's time
            "eval_overhead_at_eval_every": round((min(with_eval) - min(plain)) / min(plain), 4),
            "eval_share_of_run_at_eval_every": round((min(with_eval) - min(plain)) / min(with_eval), 4),
            "eval_overhead_at_eval_every_250": round(eval_ms / (250 * step_ms), 4),
            "eval_share_of_run_at_eval_every_250": round(eval_ms / (250 * step_ms + eval_ms), 4)}


def main(argv=None) -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args(argv)
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("eval_bench.py needs a GPU")
    c = card()
    print(f"card: {c['name']}, power limit {c['power_limit']}, max SM clock {c['max_sm_clock']}", flush=True)
    res = {"card": c, "gpus": 1, "head": bench_head(args.iters, args.rounds)}
    print(json.dumps(res["head"]), flush=True)
    res["forward"] = bench_forward(max(5, args.iters // 5), args.rounds)
    print(json.dumps(res["forward"]), flush=True)
    res["step"] = bench_step(args.rounds)
    print(json.dumps(res["step"]), flush=True)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "eval_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
