"""Pre-warmed worker process ("zygote").

Spawn -> Running of a replica is dominated by the interpreter start and ``import torch`` (seconds), not by the
control plane (milliseconds; SURVEY.md §7.3 item 1 "warm worker pool").  The node agent therefore keeps a few of
these processes parked: interpreter up, torch / torch.distributed / the worker runtime imported.  On a GPU box each
parked interpreter is pinned to one GPU slot (``CUDA_VISIBLE_DEVICES`` set when it is spawned, ``--cuda``) and also
holds a live CUDA context with the cuBLAS / cuDNN handles created; it is only handed to a container scheduled onto
that slot.  Without ``--cuda`` no CUDA call is made (the device is only known at assignment).  When a pod whose
container command is
``python -m <module> ...`` (or ``python <script> ...``) is started, the agent re-keys one parked process as that
container and sends it the assignment -- argv, environment, cwd, log file, CPU set -- over a FIFO.  The process
then *becomes* the container: same PID, supervised by the same C++ supervisor, exit status reported the usual way.

The reference has no counterpart: kubelet always starts a fresh container (pkg/controller/pod.go:528 builds the
env once at pod creation); this only removes start-up latency, the observable pod lifecycle is unchanged.

Protocol: ``python -m trainingjob_operator_b200.runtime.zygote <fifo> [--cuda]``; after the imports the zygote creates
``<fifo>.ready`` and blocks opening the FIFO.  One JSON object arrives:
``{"argv": [...], "env": {...}, "cwd": "", "log": "/path", "cpus": [..]}``.
"""
from __future__ import annotations

import json
import os
import runpy
import sys


def _preload(cuda: bool = False) -> None:
    # everything a training worker imports before touching the GPU; CUDA is initialised only when this
    # interpreter was pinned to a GPU slot at spawn time
    import numpy  # noqa: F401
    import torch  # noqa: F401
    import torch.distributed  # noqa: F401
    import torch.nn.functional  # noqa: F401

    for mod in ("trainingjob_operator_b200.runtime.worker", "trainingjob_operator_b200.runtime.trainer",
                "trainingjob_operator_b200.runtime.elastic", "trainingjob_operator_b200.models.gpt2",
                "trainingjob_operator_b200.models.bert", "trainingjob_operator_b200.parallel.ddp",
                "trainingjob_operator_b200.parallel.symm", "trainingjob_operator_b200.ops.functional"):
        try:
            __import__(mod)
        except Exception:  # noqa: BLE001 - optional pieces must not keep the pool from warming
            pass
    if cuda and torch.cuda.is_available():
        try:
            from trainingjob_operator_b200.ops import lib as _lib

            _lib.load(build_if_missing=False)                              # dlopen + module load of the sm_90a kernels
        except Exception:  # noqa: BLE001
            pass
        try:
            dev = torch.device("cuda", int(os.environ.get("AITJ_ZYGOTE_DEVICE", "0")))
            torch.cuda.set_device(dev)
            a = torch.randn(64, 64, device=dev, dtype=torch.bfloat16)
            (a @ a).sum().item()                                           # context + cuBLAS handle
            x = torch.randn(1, 8, 16, 16, device=dev, dtype=torch.bfloat16).contiguous(memory_format=torch.channels_last)
            torch.nn.functional.conv2d(x, torch.randn(8, 8, 3, 3, device=dev, dtype=torch.bfloat16), padding=1).sum().item()
            del a, x
            torch.cuda.empty_cache()
        except Exception:  # noqa: BLE001
            pass


def split_python_command(argv):
    """(kind, target, rest) for ``python [-u] -m mod args`` / ``python [-u] script.py args``; None if not python."""
    if not argv:
        return None
    exe = os.path.basename(argv[0])
    if not exe.startswith("python"):
        return None
    i = 1
    while i < len(argv) and argv[i] in ("-u", "-B", "-E", "-s"):
        i += 1
    if i >= len(argv):
        return None
    if argv[i] == "-m":
        if i + 1 >= len(argv):
            return None
        return "module", argv[i + 1], list(argv[i + 2:])
    if argv[i].startswith("-"):
        return None          # -c, -X ...: not worth emulating
    return "script", argv[i], list(argv[i + 1:])


def become(assign: dict) -> None:
    """Turn this process into the assigned container."""
    log = assign.get("log")
    if log:
        fd = os.open(log, os.O_WRONLY | os.O_CREAT | os.O_APPEND, 0o644)
        sys.stdout.flush()
        sys.stderr.flush()
        os.dup2(fd, 1)
        os.dup2(fd, 2)
        os.close(fd)
    env = assign.get("env") or {}
    os.environ.clear()
    os.environ.update({str(k): str(v) for k, v in env.items()})
    for entry in reversed([e for e in env.get("PYTHONPATH", "").split(os.pathsep) if e]):
        if entry not in sys.path:
            sys.path.insert(1, entry)       # the container's PYTHONPATH was not known when this interpreter started
    cwd = assign.get("cwd")
    if cwd:
        os.chdir(cwd)
    cpus = assign.get("cpus") or []
    if cpus:
        try:
            os.sched_setaffinity(0, set(int(c) for c in cpus))
        except OSError:
            pass
    parsed = split_python_command(assign["argv"])
    if parsed is None:
        os.execvpe(assign["argv"][0], assign["argv"], os.environ)     # not a python command after all
    kind, target, rest = parsed
    if kind == "module":
        sys.argv = [target] + rest
        sys.modules.pop(target, None)       # preloaded for its imports; run it fresh as __main__
        runpy.run_module(target, run_name="__main__", alter_sys=True)
    else:
        sys.argv = [target] + rest
        sys.path.insert(0, os.path.dirname(os.path.abspath(target)))
        runpy.run_path(target, run_name="__main__")


def main() -> int:
    fifo = sys.argv[1]
    _preload(cuda="--cuda" in sys.argv[2:])
    with open(fifo + ".ready", "w") as f:
        f.write(str(os.getpid()))
    with open(fifo, "r") as f:          # blocks until the agent opens the write end
        line = f.readline()
    try:
        os.unlink(fifo)
        os.unlink(fifo + ".ready")
    except OSError:
        pass
    if not line.strip():
        return 0                        # pool shut down without an assignment
    become(json.loads(line))
    return 0


if __name__ == "__main__":
    sys.exit(main())
