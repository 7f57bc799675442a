"""In-tree build of the sm_90a (H100) kernel library and the native control-plane core.

Two artefacts, both left next to their sources inside the package, so the package runs from the source tree:

* ``ops/libaitj_kernels.so``  -- every ``ops/csrc/*.cu`` compiled by ``nvcc`` for
  ``compute_90a/sm_90a`` with ``-lineinfo`` (plain C ABI, loaded through ``ctypes``; no
  dependency on torch's C++ ABI, so a rebuild takes seconds).
* ``core/_aitj_core*.so``     -- the C++17 control-plane runtime (work-queue, object store,
  process supervisor) as a pybind11 module.

nvcc cross-compiles without a GPU, so this is also the CPU-side "does it build" check
(``__graft_entry__.build``).
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
import sysconfig
from pathlib import Path

PKG = Path(__file__).resolve().parent.parent
OPS_DIR = PKG / "ops"
CSRC = OPS_DIR / "csrc"
CORE_DIR = PKG / "core"
KERNEL_LIB = OPS_DIR / "libaitj_kernels.so"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC",
    "-Xptxas", "-v",
]


def _nvcc() -> str | None:
    cand = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    return cand if os.path.exists(cand) else None


def _digest(paths) -> str:
    h = hashlib.sha256()
    for p in sorted(paths):
        h.update(p.name.encode())
        h.update(p.read_bytes())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build_kernels(force: bool = False, verbose: bool = False) -> Path:
    """Compile ops/csrc/*.cu into ops/libaitj_kernels.so (sm_90a)."""
    sources = sorted(CSRC.glob("*.cu"))
    headers = sorted(CSRC.glob("*.cuh"))
    stamp = OPS_DIR / ".kernels.sha256"
    digest = _digest(sources + headers)
    if not force and KERNEL_LIB.exists() and stamp.exists() and stamp.read_text() == digest:
        return KERNEL_LIB
    nvcc = _nvcc()
    if nvcc is None:
        raise RuntimeError("nvcc not found; cannot build sm_90a kernels")
    objs = []
    build_dir = OPS_DIR / "build"
    build_dir.mkdir(exist_ok=True)
    procs = []
    for src in sources:
        obj = build_dir / (src.stem + ".o")
        objs.append(obj)
        cmd = [nvcc, *NVCC_FLAGS, "-c", str(src), "-o", str(obj)]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    log = []
    for src, p in procs:
        out, _ = p.communicate()
        log.append(f"== {src.name}\n{out}")
        if p.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{out}")
    (build_dir / "ptxas.log").write_text("\n".join(log))
    if verbose:
        print("\n".join(log))
    cmd = [nvcc, "-shared", "-o", str(KERNEL_LIB), *map(str, objs), "-lcudart"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    stamp.write_text(digest)
    return KERNEL_LIB


def core_lib_path() -> Path:
    suffix = sysconfig.get_config_var("EXT_SUFFIX") or ".so"
    return CORE_DIR / f"_aitj_core{suffix}"


def build_core(force: bool = False, verbose: bool = False) -> Path:
    """Compile core/csrc/*.cpp into the pybind11 module core/_aitj_core*.so."""
    import pybind11

    sources = sorted((CORE_DIR / "csrc").glob("*.cpp"))
    headers = sorted((CORE_DIR / "csrc").glob("*.h"))
    out = core_lib_path()
    stamp = CORE_DIR / ".core.sha256"
    digest = _digest(sources + headers)
    if not force and out.exists() and stamp.exists() and stamp.read_text() == digest:
        return out
    if not sources:
        raise RuntimeError("no core sources")
    cxx = shutil.which("g++") or "g++"
    cmd = [
        cxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-fvisibility=hidden", "-pthread",
        f"-I{pybind11.get_include()}", f"-I{sysconfig.get_paths()['include']}",
        *map(str, sources), "-o", str(out),
    ]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if verbose or r.returncode != 0:
        print(r.stdout, r.stderr)
    if r.returncode != 0:
        raise RuntimeError(f"core build failed:\n{r.stderr}")
    stamp.write_text(digest)
    return out


def build_all(force: bool = False, verbose: bool = False) -> None:
    build_kernels(force=force, verbose=verbose)
    build_core(force=force, verbose=verbose)


if __name__ == "__main__":
    build_all(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print("built:", KERNEL_LIB, core_lib_path())
