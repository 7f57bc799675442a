"""GPU numerics of the cluster GEMM kernels at the edges of their work distribution (``ops.selfcheck`` case
``gemm_cluster``, run in its own process like the other kernel cases)."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.gpu
def test_cluster_gemm_edges():
    r = subprocess.run([sys.executable, "-m", "trainingjob_operator_b200.ops.selfcheck", "--case", "gemm_cluster"],
                       cwd=ROOT, capture_output=True, text=True, timeout=420)
    sys.stdout.write(r.stdout[-4000:])
    assert r.returncode == 0, f"selfcheck gemm_cluster failed:\n{r.stdout[-3000:]}\n{r.stderr[-1500:]}"
