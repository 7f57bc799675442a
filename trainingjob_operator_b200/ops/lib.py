"""ctypes loader for ``libaitj_kernels.so`` (the hand-written sm_90a kernels).

The library is a plain C ABI: every entry point takes raw device pointers and a CUDA stream
handle and returns 0 or a negative error code.  ``check`` turns non-zero codes into
exceptions so a missing or failing kernel is never silent (no eager fallback on a GPU box).
"""
from __future__ import annotations

import ctypes
import threading
from pathlib import Path

_LIB = None
_LOCK = threading.Lock()
import os

# AITJ_KERNEL_LIB points at an alternative build of the same kernels (A/B experiments on one box)
LIB_PATH = Path(os.environ.get("AITJ_KERNEL_LIB") or Path(__file__).resolve().parent / "libaitj_kernels.so")

# launch counter: every successful launch through `call` increments it; bench.py reports the
# delta over the timed region as "gpu_launches".
LAUNCHES = 0


class KernelError(RuntimeError):
    def __init__(self, msg: str, code: int = 0):
        super().__init__(msg)
        self.code = code


def load(build_if_missing: bool = True):
    global _LIB
    if _LIB is not None:
        return _LIB
    with _LOCK:
        if _LIB is not None:
            return _LIB
        if not LIB_PATH.exists():
            if not build_if_missing:
                raise KernelError(f"{LIB_PATH} missing; run python -m trainingjob_operator_b200.ops.build")
            from .build import build_kernels

            build_kernels()
        lib = ctypes.CDLL(str(LIB_PATH))
        _declare(lib)
        _LIB = lib
    return _LIB


def available() -> bool:
    try:
        load(build_if_missing=False)
        return True
    except Exception:
        return False


_P = ctypes.c_void_p
_I = ctypes.c_int
_L = ctypes.c_longlong
_F = ctypes.c_float

_SIGS = {
    "aitj_gemm_bf16": [_P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _P, _P, _P, _I, _I, _I, _I, _P],
    "aitj_num_sms": [],
    "aitj_attn_fwd": [_P, _P, _P, _P, _I, _I, _I, _I, _F, _P],
    "aitj_attn_bwd": [_P, _P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _F, _P],
    "aitj_gemm_set_colsum": [_P],
    "aitj_gemm_set_xent": [_P, _P, _P, _I],
    "aitj_xent_finish": [_P, _P, _P, _P, _P, _I, _I, _P],
    "aitj_layernorm_fwd": [_P, _P, _P, _P, _P, _P, _I, _I, _F, _P],
    "aitj_layernorm_bwd": [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _P],
    "aitj_layernorm_wide_fwd": [_P, _P, _P, _P, _P, _P, _I, _I, _F, _P],
    "aitj_layernorm_wide_bwd": [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _P],
    "aitj_embedding_fwd": [_P, _P, _P, _P, _I, _I, _I, _P],
    "aitj_embedding_bwd": [_P, _P, _P, _P, _I, _I, _I, _I, _P],
    "aitj_embedding3_fwd": [_P, _P, _P, _P, _P, _P, _I, _I, _I, _P],
    "aitj_embedding3_bwd": [_P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _P],
    "aitj_softmax_xent": [_P, _P, _P, _I, _I, _I, _F, _P],
    "aitj_colsum": [_P, _P, _I, _I, _I, _P],
    "aitj_qkv_gather_colsum": [_P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _P],
    "aitj_sumsq": [_P, _L, _P, _P],
    "aitj_adamw": [_P, _P, _P, _P, _P, _P, _P, _P, _L, _F, _F, _F, _F, _F, _I, _F, _F, _I, _P],
    "aitj_cast_f32_bf16": [_P, _P, _L, _P],
    "aitj_mc_push": [_P, _P, _L, _P],
    "aitj_peer_push": [_P, _P, _L, _P],
    "aitj_norm_share": [_P, _P, _I, _P],
    "aitj_adamw_set_shard": [_I, _I],
    "aitj_gemm_set_peers": [_P, _P, _P, _I],
    "aitj_fused_set_peers": [_P, _P, _P, _I],
    "aitj_gelu_fwd": [_P, _P, _L, _P],
    "aitj_gelu_bwd": [_P, _P, _P, _L, _P],
    "aitj_attention_decode": [_P, _P, _P, _P, _P, _I, _I, _I, _P],
    "aitj_embedding_decode": [_P, _P, _P, _P, _P, _I, _I, _P],
    "aitj_sample_tokens": [_P, _I, _I, _P, _P, _I, _P, _I, _I, _P, _F, _I, _L, _I, _I, _P],
    "aitj_embedding_doc_fwd": [_P, _P, _P, _P, _P, _I, _I, _I, _P],
    "aitj_choice_score": [_P, _P, _P, _I, _P, _P, _P],
}


def _declare(lib) -> None:
    for name, argtypes in _SIGS.items():
        try:
            fn = getattr(lib, name)
        except AttributeError:
            continue
        fn.argtypes = argtypes
        fn.restype = _I
    for name in dir(lib):
        pass


def declare(name: str, argtypes) -> None:
    """Register an extra entry point (used by optional kernels such as the NVLS collectives)."""
    _SIGS[name] = argtypes
    if _LIB is not None:
        fn = getattr(_LIB, name)
        fn.argtypes = argtypes
        fn.restype = _I


# Per-kernel device timing (eager launches only): ``profile_start()`` makes every ``call`` bracket its launch with CUDA
# events on the launching stream; ``profile_stop()`` returns {label: (launches, total ms)}.  GEMMs are labelled by operand
# layout (forward / dgrad / wgrad) and output kind.  (SURVEY.md §5.1: the reference has no tracing at all.)
_PROFILE = None


def profile_start() -> None:
    global _PROFILE
    _PROFILE = []


def profile_stop():
    global _PROFILE
    import torch

    torch.cuda.synchronize()
    out = {}
    for label, e0, e1 in _PROFILE or []:
        n, ms = out.get(label, (0, 0.0))
        out[label] = (n + 1, ms + e0.elapsed_time(e1))
    _PROFILE = None
    return out


def _label(name: str, args) -> str:
    if name != "aitj_gemm_bf16":
        return name[5:]
    a_mn, b_mn, flags, split_k, block_n = args[9], args[10], args[14], args[15], args[16]
    kind = "wgrad" if a_mn and b_mn else ("dgrad" if b_mn else "fwd")
    extra = "+peer" if flags & 16384 else ("+mc" if flags & 128 else ("+xent" if flags & 512 else ""))
    return f"gemm:{kind}{extra} N={args[4]} K={args[5]} bn={block_n} sk={split_k}"


def call(name: str, *args) -> int:
    global LAUNCHES
    lib = load()
    if _PROFILE is not None:
        import torch

        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        rc = getattr(lib, name)(*args)
        e1.record()
        _PROFILE.append((_label(name, args), e0, e1))
    else:
        rc = getattr(lib, name)(*args)
    if rc != 0:
        raise KernelError(f"{name} failed with code {rc}", rc)
    LAUNCHES += 1
    return rc
