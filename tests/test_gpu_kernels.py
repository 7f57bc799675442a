"""GPU numerics tests: each hand-written sm_90a kernel vs. a plain fp32 PyTorch reference.

Cases run in their own process (``ops.selfcheck``) so one trapping kernel cannot poison the
CUDA context of the others.
"""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run_case(name: str, timeout: int = 420):
    r = subprocess.run([sys.executable, "-m", "trainingjob_operator_b200.ops.selfcheck", "--case", name], cwd=ROOT,
                       capture_output=True, text=True, timeout=timeout)
    sys.stdout.write(r.stdout[-4000:])
    sys.stderr.write(r.stderr[-2000:])
    assert r.returncode == 0, f"selfcheck {name} failed:\n{r.stdout[-3000:]}\n{r.stderr[-1500:]}"


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["gemm_tn", "gemm_nn", "gemm_tt", "gemm_epilogue", "gemm_2cta", "gemm_quad", "graph_step", "fused_ops", "attention", "attention_bwd",
                                  "gpt2_engine", "bert_engine"])
def test_kernel_numerics(case):
    _run_case(case)


@pytest.mark.gpu
def test_kernel_library_is_loaded_not_a_fallback():
    import torch

    from trainingjob_operator_b200.ops import functional as F
    from trainingjob_operator_b200.ops import lib

    lib.load(build_if_missing=False)
    a = torch.randn(256, 128, device="cuda").bfloat16()
    b = torch.randn(256, 128, device="cuda").bfloat16()
    out = torch.empty(256, 256, device="cuda", dtype=torch.bfloat16)
    before = lib.LAUNCHES
    F.gemm(a, b, out)
    torch.cuda.synchronize()
    assert lib.LAUNCHES == before + 1
    maps = open("/proc/self/maps").read()
    assert "libaitj_kernels.so" in maps


@pytest.mark.gpu
def test_graft_smoke():
    import __graft_entry__ as g

    g.smoke()


@pytest.mark.gpu
@pytest.mark.parametrize("model,batch", [("mnist", 64), ("resnet50", 8), ("bert", 2), ("gpt2-tiny", 4)])
def test_worker_models_train_one_gpu(model, batch, tmp_path):
    """Every benchmark model runs through the worker runtime on one GPU and reports a finite, device-timed result."""
    import json

    res = str(tmp_path / "r.json")
    env = dict(os.environ, WORLD_SIZE="1", RANK="0", PYTHONPATH=ROOT)
    env.pop("AITJ_MASTER", None)
    r = subprocess.run([sys.executable, "-m", "trainingjob_operator_b200.runtime.worker", "--model", model, "--batch",
                        str(batch), "--seq", "128", "--steps", "4", "--warmup", "3", "--result", res], cwd=ROOT, env=env,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    out = json.load(open(res))
    assert out["samples_per_sec"] > 0 and out["loss_last"] == out["loss_last"]
    if model in ("bert", "gpt2-tiny"):
        assert out["gpu_launches"] > 0 and out["cuda_graph"]


@pytest.mark.gpu
def test_e2e_job_on_gpu_through_the_control_plane(tmp_path):
    """apply(AITrainingJob) -> operator -> agent -> worker pinned to GPU 0 -> Succeed, metrics reported on the job."""
    import json

    from trainingjob_operator_b200.cmd.local import LocalCluster

    worker = [sys.executable, "-m", "trainingjob_operator_b200.runtime.worker", "--model", "gpt2-tiny", "--batch", "4",
              "--seq", "128", "--steps", "5", "--warmup", "3"]
    job = {"apiVersion": "elasticdeeplearning.ai/v1", "kind": "AITrainingJob", "metadata": {"name": "gpu-e2e"},
           "spec": {"frameworkType": "pytorch", "replicaSpecs": {"trainer": {"replicas": 1, "template": {"spec": {
               "containers": [{"name": "aitj-trainer", "command": worker, "workingDir": ROOT,
                               "env": [{"name": "PYTHONPATH", "value": ROOT}],
                               "resources": {"limits": {"nvidia.com/gpu": 1}}}]}}}}}}
    with LocalCluster(num_gpus=1, workdir=str(tmp_path)) as lc:
        lc.apply(job)
        final = lc.wait_for_phase("gpu-e2e", ("Succeed", "Failed"), timeout=300)
        logs = ""
        if final.status.phase != "Succeed":
            for fn in os.listdir(os.path.join(lc.workdir, "logs")):
                logs += open(os.path.join(lc.workdir, "logs", fn)).read()[-2000:]
        assert final.status.phase == "Succeed", logs
        m = json.loads(final.annotations["aitj.b200/metrics"])
        assert m["samples_per_sec"] > 0 and m["gpu_launches"] > 0


@pytest.mark.gpu
@pytest.mark.gpu2
def test_fused_gemm_allreduce_matches_nccl_sum_on_two_gpus():
    """tools/ddp_check.py on two GPUs: the owner-sharded gradient path (wgrad GEMM epilogue -> reduce-scatter to the owner
    over NVLink peer memory, sharded AdamW, multicast all-gather) and the round-1 multicast all-reduce path against local
    gradients + NCCL all-reduce."""
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                        "--master-addr", "127.0.0.1", "--master-port", "29571", os.path.join(ROOT, "tools", "ddp_check.py")],
                       cwd=ROOT, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert '"ok": true' in r.stdout
