"""Score a GPT-2 worker's checkpoint on HellaSwag: the fp32 master weights are loaded into an engine, its bf16 compute
copy is built, and the file's completions are packed and scored as a worker scores them.  One JSON line on stdout:
``{"correct", "examples", "acc"}``.

    python -m trainingjob_operator_b200.cmd.hellaswag --model gpt2 --ckpt PATH --data hellaswag_val.bin
        [--batch 16 --seq 1024]

The file is llm.c's eval file (``dev/data/hellaswag.py``).  With the ``--batch`` and ``--seq`` of a worker, on the
checkpoint of a step the worker scored, it prints that step's ``hellaswag`` record: same packing, same kernels.
"""
from __future__ import annotations

import argparse
import json
import sys

import torch

from ..models.gpt2 import GPT2_MODELS


def parse_args(argv=None):
    ap = argparse.ArgumentParser(prog="aitj-hellaswag")
    ap.add_argument("--model", default="gpt2", choices=list(GPT2_MODELS))
    ap.add_argument("--ckpt", required=True, metavar="PATH", help="a worker checkpoint (--ckpt-dir)")
    ap.add_argument("--data", required=True, metavar="PATH", help="llm.c's HellaSwag eval file")
    ap.add_argument("--batch", type=int, default=16, help="rows per micro-batch")
    ap.add_argument("--seq", type=int, default=1024, help="positions per row, a multiple of 128")
    ap.add_argument("--cpu", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args(argv)
    if args.batch < 1:
        ap.error(f"--batch {args.batch}: at least one row")
    if args.seq < 128 or args.seq % 128:
        ap.error(f"--seq must be a positive multiple of 128 (the document-masked attention's tile), not {args.seq}")
    return args


def main(argv=None, out=None) -> int:
    from ..models.gpt2 import GPT2Engine, gpt2_config
    from ..runtime.checkpoint import load_into
    from ..runtime.hellaswag import HellaSwagData
    from ..runtime.trainer import EngineTrainer

    args = parse_args(argv)
    out = out or sys.stdout
    cfg = gpt2_config(args.model)
    seq = min(args.seq, cfg.block_size)
    if args.cpu:
        device = torch.device("cpu")
    else:
        if not torch.cuda.is_available():
            raise SystemExit("scoring needs a CUDA device (hand-written sm_90a kernels)")
        device = torch.device("cuda", torch.cuda.current_device())
    data = HellaSwagData(args.data, cfg.vocab_size, args.batch, seq, pin=device.type == "cuda")
    eng = GPT2Engine(cfg, args.batch, seq, device)
    if load_into(args.ckpt, eng.params.state_tensors()) is None:
        raise SystemExit(f"no checkpoint at {args.ckpt}")
    eng.params.refresh_compute_copy()
    trainer = EngineTrainer(eng, use_graph=False)
    correct, examples = trainer.score(data.inputs(k) for k in range(data.micro_batches))
    out.write(json.dumps({"correct": correct, "examples": examples, "acc": correct / examples}) + "\n")
    out.flush()
    return 0


if __name__ == "__main__":
    sys.exit(main())
