"""HellaSwag scoring on one H100: what packing the completions as documents saves, and what an evaluation costs.

    python tools/hellaswag_bench.py --out DIR [--examples 10042] [--ctx 20 80] [--end 5 40] [--models gpt2,gpt2-xl]
        [--batch 16] [--seq 1024] [--rounds 3] [--iters 20]

A seeded synthetic file in llm.c's format holds ``--examples`` examples (10042, the size of HellaSwag's validation set)
whose context and ending lengths are drawn uniformly from ``--ctx`` and ``--end``; the real set's length distribution
is not used.  For each model, with random weights at B x T:

* host: the packer's micro-batch count and row fill (share of positions holding a completion), and the micro-batch
  count of one completion per row, ceil(4E / B), for comparison;
* device (CUDA events, after warm-up, ``--rounds`` times): one whole evaluation (``EngineTrainer.score`` over every
  micro-batch), and ``score_forward`` against ``eval_forward`` on one micro-batch, ``--iters`` launches each, alternating.

The speed-up of packing over one completion per row is DERIVED from the micro-batch counts and the measured time per
micro-batch; it is not measured.  Prints the card and its power limit and writes ``DIR/hellaswag_bench.json``.
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


def synthetic_file(path, n, ctx, end, vocab, seed):
    import numpy as np

    from trainingjob_operator_b200.runtime.hellaswag import write_examples

    rng = np.random.default_rng(seed)
    exs = []
    for _ in range(n):
        c = rng.integers(0, vocab, int(rng.integers(ctx[0], ctx[1] + 1)))
        ends = [rng.integers(0, vocab, int(rng.integers(end[0], end[1] + 1))) for _ in range(4)]
        exs.append((int(rng.integers(0, 4)), c, ends))
    return write_examples(path, exs)


def _time(fn, iters):
    import torch

    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / iters


def bench_model(name, path, B, T, rounds, iters):
    import torch

    from trainingjob_operator_b200.models.gpt2 import GPT2Engine, gpt2_config
    from trainingjob_operator_b200.runtime.hellaswag import HellaSwagData
    from trainingjob_operator_b200.runtime.trainer import EngineTrainer

    cfg = gpt2_config(name)
    data = HellaSwagData(path, cfg.vocab_size, B, T, pin=True)
    E, K = data.examples, data.micro_batches
    one_per_row = -(-4 * E // B)
    eng = GPT2Engine(cfg, B, T, "cuda", seed=0)
    tr = EngineTrainer(eng, use_graph=False)

    def evaluation():
        return tr.score(data.inputs(k) for k in range(K))

    # one micro-batch of the file for the per-forward arms; eval_forward reads the same tokens and targets
    tok, tgt, ds, spans, labels = data.inputs(0)
    spans_d, labels_d = spans.cuda(), labels.cuda()

    def load():
        eng.tok.copy_(tok, non_blocking=True)
        eng.tgt.copy_(tgt, non_blocking=True)

    def score():
        eng.score_forward(ds, spans_d, labels_d, spans.shape[0])

    def ev():
        eng.eval_forward()

    result = evaluation()                      # warm-up: every kernel and shape of the evaluation
    load()
    for fn in (score, ev):
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    t_eval, t_score, t_ev = [], [], []
    for _ in range(rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        again = evaluation()
        e1.record()
        e1.synchronize()
        assert again == result, (again, result)
        t_eval.append(e0.elapsed_time(e1))
        load()
        t_score.append(_time(score, iters))
        t_ev.append(_time(ev, iters))
    ms_eval = min(t_eval)
    per_micro = ms_eval / K
    out = {
        "model": name, "batch": B, "seq": T, "examples": E, "correct": result[0],
        "host": {"micro_batches_packed": K, "row_fill_packed": round(data.fill, 4),
                 "micro_batches_one_completion_per_row": one_per_row,
                 "micro_batch_ratio": round(one_per_row / K, 2)},
        "device": {"ms_per_evaluation": round(ms_eval, 2), "ms_per_evaluation_rounds": [round(t, 2) for t in t_eval],
                   "ms_per_micro_batch_in_evaluation": round(per_micro, 3),
                   "ms_score_forward": round(min(t_score), 3), "ms_score_forward_rounds": [round(t, 3) for t in t_score],
                   "ms_eval_forward": round(min(t_ev), 3), "ms_eval_forward_rounds": [round(t, 3) for t in t_ev]},
        "derived_not_measured": {
            "ms_per_evaluation_one_completion_per_row": round(per_micro * one_per_row, 1),
            "speedup_of_packing": round(one_per_row / K, 2),
            "how": "one completion per row would run ceil(4E / B) micro-batches at the measured time per micro-batch"},
    }
    del tr, eng
    torch.cuda.empty_cache()
    return out


def main(argv=None) -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--examples", type=int, default=10042)
    ap.add_argument("--ctx", type=int, nargs=2, default=(20, 80), metavar=("MIN", "MAX"), help="context tokens")
    ap.add_argument("--end", type=int, nargs=2, default=(5, 40), metavar=("MIN", "MAX"), help="ending tokens")
    ap.add_argument("--models", default="gpt2,gpt2-xl")
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--seq", type=int, default=1024)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args(argv)
    os.makedirs(a.out, exist_ok=True)
    import tempfile

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("hellaswag_bench measures on a CUDA device")
    dev = card()
    print(f"card: {dev}", flush=True)
    with tempfile.TemporaryDirectory() as tmp:
        path = synthetic_file(os.path.join(tmp, "hellaswag_synthetic.bin"), a.examples, a.ctx, a.end, 50257, a.seed)
        res = {"card": dev, "file": {"examples": a.examples, "ctx_tokens": list(a.ctx), "end_tokens": list(a.end),
                                     "seed": a.seed, "lengths": "uniform, synthetic (not HellaSwag's distribution)"},
               "models": []}
        for name in a.models.split(","):
            r = bench_model(name, path, a.batch, a.seq, a.rounds, a.iters)
            print(json.dumps(r), flush=True)
            res["models"].append(r)
    res["card_after"] = card()
    with open(os.path.join(a.out, "hellaswag_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
