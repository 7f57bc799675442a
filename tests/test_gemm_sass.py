"""What ptxas made of the wgmma GEMM's main loop, checked without a GPU.

A GPU-scope memory fence between two batches of tensor-core instructions stalls the whole consumer warpgroup (wgmma is
warpgroup-collective).  An mbarrier arrive with .release.cluster semantics compiles to such a fence on sm_90a, so a
ring stage handed back that way costs one per k-block and CTA of the cluster.  This compiles ``gemm_wgmma.cu`` for
sm_90a and requires that no ``MEMBAR.*.GPU`` lies between the first and the last HGMMA of any GEMM instantiation.
"""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "trainingjob_operator_b200", "ops", "csrc", "gemm_wgmma.cu")


def _tool(name):
    path = shutil.which(name) or os.path.join("/usr/local/cuda/bin", name)
    return path if os.path.exists(path) else None


@pytest.fixture(scope="module")
def gemm_sass(tmp_path_factory):
    nvcc, cuobjdump = _tool("nvcc"), _tool("cuobjdump")
    if not nvcc or not cuobjdump:
        pytest.skip("needs nvcc and cuobjdump")
    cubin = str(tmp_path_factory.mktemp("sass") / "gemm.cubin")
    subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-cubin", SRC, "-o", cubin],
                   check=True, capture_output=True, text=True, timeout=900)
    out = subprocess.run([cuobjdump, "-sass", cubin], check=True, capture_output=True, text=True).stdout
    funcs, cur = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            funcs[cur] = []
        elif cur is not None and re.search(r"/\*[0-9a-f]{4,}\*/", line):
            funcs[cur].append(line)
    return {k: v for k, v in funcs.items() if "gemm_bf16_wgmma_kernel" in k}


def test_every_layout_and_cluster_size_is_instantiated(gemm_sass):
    # 4 operand layouts x (2-CTA and 4-CTA clusters + the 1-CTA tiles)
    assert len(gemm_sass) >= 12, sorted(gemm_sass)


def test_no_gpu_scope_fence_inside_the_main_loop(gemm_sass):
    """The main loop's body is laid out once, with its stage releases after the last HGMMA, so every fence after the
    first HGMMA counts -- except the one of the cluster barrier at kernel exit (MEMBAR then UCGABAR_ARV)."""
    bad = {}
    for name, lines in gemm_sass.items():
        mma = [i for i, s in enumerate(lines) if "HGMMA" in s]
        assert mma, f"{name}: no HGMMA"
        fences = [lines[i].split("*/")[1].strip() for i in range(mma[0], len(lines))
                  if re.search(r"MEMBAR\S*\.GPU", lines[i]) and not any("UCGABAR_ARV" in s for s in lines[i:i + 5])]
        if fences:
            bad[name] = fences
    assert not bad, "GPU-scope fences after the first HGMMA:\n" + "\n".join(f"{k}: {len(v)} x {v[0]}" for k, v in bad.items())
