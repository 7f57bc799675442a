"""Document-masked attention on one H100: kernel times of the masked wgmma flash attention against the causal kernels on
several document layouts, and the worker's step time when it trains on a token shard.

    python tools/doc_attention_bench.py --out DIR [--iters 50] [--steps 30] [--repeats 2] [--skip-train]

Prints the card and its power limit and writes ``DIR/doc_attention_bench.json``.  Kernel times are CUDA-event times over
``--iters`` launches after a warm-up, at B16 T1024 H12 (GPT-2 small).  For every layout it also reports the key blocks
the kernels visit, counted on the host from ``doc_start`` (forward: 64-key blocks per 128-row query tile; backward:
64-query blocks per 64-key block), next to the causal count; TFLOP/s count the visible score elements only (forward
4*64 FLOP each, backward 10*64).  The training runs alternate three worker configurations on one generated shard
(``--data`` with the default cuDNN attention, ``--data --doc-mask``, ``--data`` with AITJ_ATTN=AITJ_ATTN_BWD=wgmma) and
repeat each ``--repeats`` times.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = [x.strip() for x in r.stdout.splitlines()[0].split(",")]
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def layouts(T, seed=0):
    """name -> per-row document lengths generator (each row gets its own draw for the random layout)."""
    from trainingjob_operator_b200.ops.selfcheck import doc_start_from_lengths

    rng = np.random.default_rng(seed)

    def rand_row():
        lens, n = [], 0
        while n < T:
            lens.append(int(max(1, rng.exponential(256))))
            n += lens[-1]
        return doc_start_from_lengths(lens, T)

    return {"one_doc": lambda: doc_start_from_lengths([T], T),
            "fixed_512": lambda: doc_start_from_lengths([512], T),
            "fixed_128": lambda: doc_start_from_lengths([128], T),
            "fixed_32": lambda: doc_start_from_lengths([32], T),
            "random_mean_256": rand_row}


def blocks_visited(ds_row, T):
    """(forward key blocks, backward query blocks, visible score elements) of one sequence."""
    ds = np.asarray(ds_row)
    fwd = sum((q0 + 128) // 64 - min(max(int(ds[q0]), 0), q0) // 64 for q0 in range(0, T, 128))
    bwd = 0
    for kv0 in range(0, T, 64):
        last = kv0 + 63
        qe = last + 1
        while qe < T and ds[qe] <= last:
            qe += 1
        bwd += max((qe + 63) // 64, kv0 // 64 + 1) - kv0 // 64
    visible = int(sum(q - ds[q] + 1 for q in range(T)))
    return fwd, bwd, visible


def kernel_bench(iters):
    import torch

    from trainingjob_operator_b200.ops import functional as F

    B, T, H = 16, 1024, 12
    C = H * 64
    torch.manual_seed(0)
    qkv = torch.randn(B * T, 3 * C, device="cuda").bfloat16()
    d_out = torch.randn(B * T, C, device="cuda").bfloat16()
    out = torch.empty(B * T, C, device="cuda", dtype=torch.bfloat16)
    lse = torch.empty(B, H, T, device="cuda")
    delta = torch.empty(B, H, T, device="cuda")
    dq_acc = torch.zeros(B * T, C, device="cuda")
    d_qkv = torch.empty_like(qkv)

    def timeit(fn):
        for _ in range(5):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / iters * 1e3

    def run(ds):
        fwd = lambda: F.attention_fwd(qkv, out, lse, B, T, H, causal=True, doc_start=ds)  # noqa: E731

        def both():
            fwd()
            F.attention_bwd(qkv, out, d_out, lse, delta, dq_acc, d_qkv, B, T, H, causal=True, doc_start=ds)

        return timeit(fwd), timeit(both)

    causal_fb = blocks_visited(np.zeros(T, dtype=np.int32), T)
    rows = []
    lay = layouts(T)
    configs = [("causal (unmasked kernels)", None)] + [(n, torch.cat([g() for _ in range(B)])) for n, g in lay.items()]
    # two rounds, alternating the layouts, so that a drift of the card shows as a spread between the rounds
    times = {n: [] for n, _ in configs}
    for _ in range(2):
        for name, ds in configs:
            times[name].append(run(ds.cuda() if ds is not None else None))
    for name, ds in configs:
        if ds is None:
            fb = (causal_fb[0] * B, causal_fb[1] * B, causal_fb[2] * B)
        else:
            per = [blocks_visited(ds[b * T:(b + 1) * T].numpy(), T) for b in range(B)]
            fb = tuple(sum(p[i] for p in per) for i in range(3))
        t_f = min(t[0] for t in times[name])
        t_fb = min(t[1] for t in times[name])
        vis = fb[2] * H
        rows.append({"layout": name, "fwd_us": round(t_f, 2), "fwd_bwd_us": round(t_fb, 2),
                     "fwd_us_rounds": [round(t[0], 2) for t in times[name]],
                     "fwd_bwd_us_rounds": [round(t[1], 2) for t in times[name]],
                     "fwd_key_blocks": fb[0] * H, "bwd_query_blocks": fb[1] * H,
                     "causal_fwd_key_blocks": causal_fb[0] * B * H, "causal_bwd_query_blocks": causal_fb[1] * B * H,
                     "visible_scores": vis,
                     "fwd_tflops_visible": round(4 * 64 * vis / t_f / 1e6, 1),
                     "fwd_bwd_tflops_visible": round(14 * 64 * vis / t_fb / 1e6, 1)})
        print(json.dumps(rows[-1]), flush=True)
    return rows


def write_shard(path, n_tokens, seed=0):
    """A GPT-2-vocabulary shard in llm.c format: documents of exponentially distributed length (mean 256), each opened
    by the end-of-text token."""
    rng = np.random.default_rng(seed)
    toks = rng.integers(0, 50256, n_tokens).astype(np.uint16)
    pos = 0
    while pos < n_tokens:
        toks[pos] = 50256
        pos += int(max(1, rng.exponential(256)))
    hdr = np.zeros(256, dtype="<i4")
    hdr[0], hdr[1], hdr[2] = 20240520, 1, n_tokens
    with open(path, "wb") as f:
        f.write(hdr.tobytes())
        f.write(toks.tobytes())


def train_bench(steps, warmup, repeats, tmp):
    shard = os.path.join(tmp, "bench_000.bin")
    write_shard(shard, (steps + warmup + 4) * 16 * 1024 + 1)
    arms = [("data (cuDNN attention)", [], {}),
            ("data + doc-mask (wgmma attention, masked)", ["--doc-mask"], {}),
            ("data + wgmma attention (unmasked)", [], {"AITJ_ATTN": "wgmma", "AITJ_ATTN_BWD": "wgmma"})]
    out = {name: [] for name, _, _ in arms}
    for rep in range(repeats):
        for name, extra, env_extra in arms:
            res = os.path.join(tmp, "r.json")
            env = dict(os.environ, WORLD_SIZE="1", RANK="0", PYTHONPATH=ROOT, **env_extra)
            for k in ("AITJ_MASTER", "AITJ_ATTN", "AITJ_ATTN_BWD"):
                if k not in env_extra:
                    env.pop(k, None)
            r = subprocess.run([sys.executable, "-m", "trainingjob_operator_b200.runtime.worker", "--model", "gpt2",
                                "--batch", "16", "--seq", "1024", "--steps", str(steps), "--warmup", str(warmup),
                                "--data", shard, "--result", res] + extra, cwd=ROOT, env=env, capture_output=True,
                               text=True, timeout=900)
            if r.returncode != 0:
                raise RuntimeError(f"{name}: worker failed\n{r.stdout[-2000:]}\n{r.stderr[-3000:]}")
            j = json.load(open(res))
            out[name].append({"ms_per_step": round(j["ms_per_step"], 3), "loss_last": j["loss_last"],
                              "cuda_graph": j["cuda_graph"]})
            print(f"[train] {name} run {rep}: {j['ms_per_step']:.2f} ms/step loss {j['loss_last']:.3f}", flush=True)
    return out


def main(argv=None) -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--skip-train", action="store_true")
    args = ap.parse_args(argv)
    import torch

    if not torch.cuda.is_available():
        print("no CUDA device: nothing measured", file=sys.stderr)
        return 2
    result = {"card": card(), "shape": "B16 T1024 H12 D64", "iters": args.iters}
    print(json.dumps(result["card"]), flush=True)
    result["kernels"] = kernel_bench(args.iters)
    if not args.skip_train:
        with tempfile.TemporaryDirectory() as tmp:
            result["train_gpt2_small_b16_t1024"] = train_bench(args.steps, args.warmup, args.repeats, tmp)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "doc_attention_bench.json"), "w") as f:
        json.dump(result, f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
