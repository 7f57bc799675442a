"""Generate text from a GPT-2 worker's checkpoint: the fp32 master weights are loaded into an engine, its bf16 compute
copy is built, and ``models.generate.GPT2Generator`` samples from it.  One JSON line per sequence on stdout.

    python -m trainingjob_operator_b200.cmd.generate --model gpt2 --ckpt PATH [--prompt IDS] [--tokens K] [--count S]
        [--temperature T] [--top-k K] [--seed N] [--tokenizer PATH]

A worker reports the seed of each of its generations (``generations[].seed`` in its result): passed as ``--seed``, with
that generation's prompt, count and sampling settings, on the checkpoint of the same step, it gives the same tokens.
"""
from __future__ import annotations

import argparse
import json
import sys

import torch

from ..models.gpt2 import GPT2_MODELS


def parse_args(argv=None):
    ap = argparse.ArgumentParser(prog="aitj-generate")
    ap.add_argument("--model", default="gpt2", choices=list(GPT2_MODELS))
    ap.add_argument("--ckpt", required=True, metavar="PATH", help="a worker checkpoint (--ckpt-dir)")
    ap.add_argument("--prompt", default=None, metavar="IDS", help="comma-separated token ids (default: --eot-token)")
    ap.add_argument("--eot-token", type=int, default=50256)
    ap.add_argument("--tokens", type=int, default=64, metavar="K", help="new tokens per sequence")
    ap.add_argument("--count", type=int, default=4, metavar="S", help="sequences")
    ap.add_argument("--temperature", type=float, default=1.0, help="0 = greedy")
    ap.add_argument("--top-k", type=int, default=0, help="0 = the whole vocabulary")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--tokenizer", default="", metavar="PATH", help="an llm.c gpt2_tokenizer.bin: also print the text")
    ap.add_argument("--gemm", default="wgmma", choices=["wgmma", "cublas"])
    ap.add_argument("--no-graph", action="store_true", help="run every decode step eagerly")
    ap.add_argument("--cpu", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args(argv)
    try:
        args.prompt = [int(t) for t in args.prompt.split(",")] if args.prompt is not None else [args.eot_token]
    except ValueError:
        ap.error(f"--prompt {args.prompt!r} is not a comma-separated list of token ids")
    if args.tokens < 0 or args.count < 1 or args.top_k < 0 or not args.temperature >= 0 or args.seed < 0:
        ap.error("--tokens, --temperature, --top-k and --seed cannot be negative, and --count must be at least 1")
    return args


def main(argv=None, out=None) -> int:
    from ..models.generate import GPT2Generator
    from ..models.gpt2 import GPT2Engine, gpt2_config
    from ..runtime.checkpoint import load_into

    args = parse_args(argv)
    out = out or sys.stdout
    cfg = gpt2_config(args.model)
    tokenizer = None
    if args.tokenizer:
        from ..runtime.tokenizer import Tokenizer

        tokenizer = Tokenizer(args.tokenizer)
    if args.cpu:
        device = torch.device("cpu")
    else:
        if not torch.cuda.is_available():
            raise SystemExit("generation needs a CUDA device (hand-written sm_90a kernels)")
        device = torch.device("cuda", torch.cuda.current_device())
    # an engine of one one-token row: the generator brings its own buffers, the engine holds the weights
    eng = GPT2Engine(cfg, 1, 1, device, gemm_backend=args.gemm)
    if load_into(args.ckpt, eng.params.state_tensors()) is None:
        raise SystemExit(f"no checkpoint at {args.ckpt}")
    eng.params.refresh_compute_copy()
    gen = GPT2Generator(eng, args.count, min(cfg.block_size, len(args.prompt) + args.tokens))
    toks = gen.generate(args.prompt, args.tokens, temperature=args.temperature, top_k=args.top_k, seed=args.seed,
                        use_graph=device.type == "cuda" and not args.no_graph)
    for i, row in enumerate(toks.tolist()):
        rec = {"sequence": i, "tokens": row}
        if tokenizer is not None:
            rec["text"] = tokenizer.decode(row)
        out.write(json.dumps(rec) + "\n")
    out.flush()
    return 0


if __name__ == "__main__":
    sys.exit(main())
