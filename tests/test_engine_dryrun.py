"""The engines, the trainer and the bucketed DDP path executed on CPU with the kernel entry points emulated in plain
PyTorch (``tests/kernel_emulation.py``): what is checked is the control flow AROUND the hand-written kernels -- which the
build container can otherwise never run -- against the fp32 reference models.  The kernels themselves are checked on the
device (``tests/test_gpu_kernels.py``)."""
import os
import subprocess
import sys
import textwrap
import types

import numpy as np
import pytest
import torch

import kernel_emulation as ke

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def rel(a, b):
    return float((a.float() - b.float()).norm() / (b.float().norm() + 1e-12))


def gpt2_pair(monkeypatch, env=None, seed=3):
    from trainingjob_operator_b200.models.gpt2 import GPT2Config, GPT2Engine, GPT2Reference

    ke.install(monkeypatch)
    for k, v in (env or {}).items():
        monkeypatch.setenv(k, v)
    cfg = GPT2Config(vocab_size=1000, n_layer=2, n_head=4, n_embd=256, block_size=128, name="t")
    B, T = 2, 128
    eng = GPT2Engine(cfg, B, T, "cpu", seed=seed, gemm_backend="wgmma")
    g = torch.Generator().manual_seed(9)
    for s_ in eng.params.specs:               # biases / LayerNorm gains away from their symmetric initial values
        if len(s_.shape) == 1:
            eng.params.w32(s_.name).add_(torch.randn(s_.shape, generator=g) * 0.05)
    eng.params.refresh_compute_copy()
    ref = GPT2Reference(cfg, eng.params)
    tok = torch.randint(0, cfg.vocab_size, (B, T), generator=torch.Generator().manual_seed(5))
    tgt = torch.roll(tok, -1, dims=1)
    eng.tok.copy_(tok.view(-1))
    eng.tgt.copy_(tgt.view(-1))
    return cfg, eng, ref, tok, tgt


GPT2_GRADS = ("wte", "wpe", "h0.qkv_w", "h0.qkv_b", "h0.proj_w", "h0.proj_b", "h0.fc_w", "h0.fc_b", "h0.fc2_w",
              "h0.fc2_b", "h0.ln1_w", "h0.ln1_b", "h1.ln2_w", "h1.ln2_b", "h1.fc2_w", "h1.qkv_w", "lnf_w", "lnf_b")


# (AITJ_ATTN=wgmma with the library backward calls a cuDNN-only aten op: that combination exists on the GPU only)
@pytest.mark.parametrize("env", [{}, {"AITJ_ATTN": "wgmma", "AITJ_ATTN_BWD": "wgmma"},
                                 {"AITJ_GEMM_CFG": "fwd:768x256=256,dgrad:256x768=128,wgrad:1024x256=512/4"},
                                 {"AITJ_GEMM_PAIR": "0"}],
                         ids=["default", "attn-fwd-bwd", "gemm-table", "no-pair"])
def test_gpt2_engine_control_flow_matches_the_reference_model(monkeypatch, env):
    """Forward + backward of the explicit engine: every gradient lands in the right slice of the flat buffer with the
    right accumulate / overwrite behaviour (a wrong buffer rotation, a skipped bias gradient or a doubled accumulation
    shows as an O(1) error; bf16 storage of activations costs ~1e-2)."""
    cfg, eng, ref, tok, tgt = gpt2_pair(monkeypatch, env)
    if env.get("AITJ_ATTN"):
        assert eng.attn_impl == "wgmma" and eng.attn_bwd_impl == env.get("AITJ_ATTN_BWD", "cudnn")
    eng.params.g32.zero_()
    eng.forward()
    eng.backward()
    loss = ref(tok, tgt)
    loss.backward()
    assert abs(float(eng.loss) - float(loss.detach())) < 2e-2 * float(loss.detach())
    for name in GPT2_GRADS:
        assert rel(eng.params.grad(name), ref.p(name).grad) < 6e-2, name
    # a second backward ACCUMULATES (the optimizer sweep is what clears the buffer)
    g1 = eng.params.grad("h0.fc_w").clone()
    eng.forward()
    eng.backward()
    assert rel(eng.params.grad("h0.fc_w"), 2 * g1) < 1e-3
    if "AITJ_GEMM_CFG" in env:
        assert eng.gemm_cfg["wgrad:1024x256"] == (512, 4) and 128 in ke.CALLS["gemm_block_n"]
    if env.get("AITJ_GEMM_PAIR") == "0":
        assert 512 not in ke.CALLS["gemm_block_n"]


def test_library_gemm_arm_of_the_engine_matches_the_reference_model(monkeypatch):
    """``--gemm cublas`` (the A/B arm: library matmuls + standalone element-wise kernels instead of fused epilogues) walks
    the other branch of every GEMM front-end; same gradients."""
    from trainingjob_operator_b200.models.gpt2 import GPT2Config, GPT2Engine, GPT2Reference

    ke.install(monkeypatch)
    cfg = GPT2Config(vocab_size=1000, n_layer=2, n_head=4, n_embd=256, block_size=128, name="t")
    B, T = 2, 128
    eng = GPT2Engine(cfg, B, T, "cpu", seed=3, gemm_backend="cublas")
    ref = GPT2Reference(cfg, eng.params)
    tok = torch.randint(0, cfg.vocab_size, (B, T), generator=torch.Generator().manual_seed(5))
    tgt = torch.roll(tok, -1, dims=1)
    eng.tok.copy_(tok.view(-1))
    eng.tgt.copy_(tgt.view(-1))
    n0 = len(ke.CALLS["gemm_block_n"])
    eng.params.g32.zero_()
    eng.forward()
    eng.backward()
    assert len(ke.CALLS["gemm_block_n"]) == n0                    # no hand-written GEMM on this arm
    loss = ref(tok, tgt)
    loss.backward()
    assert abs(float(eng.loss) - float(loss.detach())) < 2e-2 * float(loss.detach())
    for name in ("wte", "wpe", "h0.qkv_w", "h0.qkv_b", "h0.proj_w", "h0.fc_w", "h0.fc_b", "h0.fc2_w", "h1.ln2_w", "lnf_b"):
        assert rel(eng.params.grad(name), ref.p(name).grad) < 6e-2, name


def test_gpt2_engine_optimizer_reduces_the_loss_and_keeps_the_compute_copy_in_sync(monkeypatch):
    cfg, eng, ref, tok, tgt = gpt2_pair(monkeypatch)
    eng.params.g32.zero_()
    eng.forward()
    l0 = float(eng.loss)
    for step in range(1, 6):
        eng.backward()
        eng.optimizer_step(lr=1e-3, step=step)
        assert float(eng.params.g32.abs().max()) == 0.0          # cleared by the sweep
        eng.forward()
    assert float(eng.loss) < l0 - 0.05, (l0, float(eng.loss))
    P = eng.params
    assert torch.equal(P.p16, P.p32.to(torch.bfloat16))          # bf16 compute copy refreshed from the master weights
    # gradient clipping: an absurd max_norm leaves the update direction, a tiny one shrinks the step
    before = P.p32.clone()
    eng.backward()
    eng.optimizer_step(lr=1e-3, step=6, max_norm=1e-6)
    small = float((P.p32 - before).abs().max())
    assert 0 < small < 2e-3


def test_bert_engine_control_flow_matches_the_reference_model(monkeypatch):
    from trainingjob_operator_b200.models.bert import BertConfig, BertEngine, BertReference, SyntheticMLM

    ke.install(monkeypatch)
    cfg = BertConfig.tiny()
    B, T = 2, 128
    eng = BertEngine(cfg, B, T, "cpu", seed=3)
    g = torch.Generator().manual_seed(9)
    for s_ in eng.params.specs:
        if len(s_.shape) == 1:
            eng.params.w32(s_.name).add_(torch.randn(s_.shape, generator=g) * 0.05)
    eng.params.w32("dec_b")[cfg.vocab_size:].zero_()
    eng.params.refresh_compute_copy()
    ref = BertReference(cfg, eng.params)
    data = SyntheticMLM(cfg.vocab_size, B, T, n_batches=1, seed=5, pin=False)
    tok, typ, lab = data.next()
    for dst, src in zip(eng.input_tensors(), (tok, typ, lab)):
        dst.copy_(src)
    assert eng.n_masked == data.n_masked
    eng.params.g32.zero_()
    eng.forward()
    eng.backward()
    loss = ref(tok.view(B, T), typ.view(B, T), lab.view(B, T))
    loss.backward()
    assert abs(float(eng.loss) - float(loss.detach())) < 2e-2 * float(loss.detach())
    for name in ("wte", "wpe", "wtt", "emb_ln_w", "emb_ln_b", "h0.qkv_w", "h0.qkv_b", "h0.proj_w", "h0.proj_b", "h0.ln1_w",
                 "h0.ln1_b", "h0.fc_w", "h0.fc_b", "h0.fc2_w", "h0.fc2_b", "h0.ln2_w", "h1.ln2_b", "h1.fc2_w", "h1.qkv_w",
                 "mlm_w", "mlm_b", "mlm_ln_w", "mlm_ln_b", "dec_b"):
        gref, got = ref.p(name).grad, eng.params.grad(name)
        if name == "dec_b":
            gref, got = gref[:cfg.vocab_size], got[:cfg.vocab_size]
        assert rel(got, gref) < 6e-2, name
    l0 = float(eng.loss)
    for step in range(1, 5):
        eng.optimizer_step(lr=1e-3, step=step)
        eng.forward()
        eng.backward()
    assert float(eng.loss) < l0


def test_engine_trainer_steps_on_cpu_and_feeds_inputs_and_schedule(monkeypatch):
    """EngineTrainer.step: host inputs -> device tensors, lr schedule into the device scalars, eager step (no CUDA graph
    off-GPU), loss read back."""
    from trainingjob_operator_b200.runtime.trainer import EngineTrainer, cosine_lr

    cfg, eng, ref, tok, tgt = gpt2_pair(monkeypatch)
    tr = EngineTrainer(eng, lr=1e-3, use_graph=True)
    assert tr.use_graph is False and tr.reducer is None and tr.allreduce_backend == "none"
    losses = [tr.step(tok.view(-1), tgt.view(-1)) for _ in range(5)]
    assert all(l == l for l in losses) and losses[-1] < losses[0]
    assert abs(float(eng.dyn[0]) - cosine_lr(5, 1e-3)) < 1e-9
    assert tr.step_count == 5


DDP_SCRIPT = """
import os, sys, json, torch, torch.distributed as dist
sys.path.insert(0, {root!r}); sys.path.insert(0, os.path.join({root!r}, "tests"))
import kernel_emulation as ke
ke.install()
from trainingjob_operator_b200.models.gpt2 import GPT2Config, GPT2Engine
from trainingjob_operator_b200.runtime.trainer import EngineTrainer
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
dist.init_process_group("gloo", rank=rank, world_size=world)
cfg = GPT2Config(vocab_size=1000, n_layer=2, n_head=4, n_embd=256, block_size=128, name="t")
eng = GPT2Engine(cfg, 2, 128, "cpu", seed=3, gemm_backend="wgmma")
tr = EngineTrainer(eng, lr=1e-3, use_graph=False, allreduce="nccl")
assert tr.reducer is not None and tr.segmented and eng.segment_join is True
g = torch.Generator().manual_seed(100 + rank)          # every rank its own data
out = {{"rank": rank, "buckets": [b[0] for b in tr.reducer.buckets], "losses": []}}
for step in range(4):
    tok = torch.randint(0, cfg.vocab_size, (2 * 128,), generator=g)
    out["losses"].append(tr.step(tok, torch.roll(tok, -1)))
p = eng.params.p32.clone()
ref = p.clone()
dist.broadcast(ref, 0)
out["max_param_diff_to_rank0"] = float((p - ref).abs().max())
out["grad_left"] = float(eng.params.g32.abs().max())
print("RESULT " + json.dumps(out), flush=True)
dist.destroy_process_group()
"""


@pytest.mark.slow
def test_bucketed_ddp_over_gloo_keeps_the_replicas_identical(tmp_path):
    """The NCCL-mode trainer (bucket hooks fired by the backward segments, join before the optimizer, gradient divided by
    the world size in the sweep) with two gloo ranks on different data: parameters stay bit-identical across ranks."""
    script = tmp_path / "ddp.py"
    script.write_text(textwrap.dedent(DDP_SCRIPT.format(root=ROOT)))
    import socket

    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    procs = []
    for r in range(2):
        env = dict(os.environ, RANK=str(r), WORLD_SIZE="2", MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port),
                   OMP_NUM_THREADS="2")
        procs.append(subprocess.Popen([sys.executable, str(script)], env=env, stdout=subprocess.PIPE,
                                      stderr=subprocess.STDOUT, text=True))
    outs = [p.communicate(timeout=600)[0] for p in procs]
    import json

    res = []
    for o, p in zip(outs, procs):
        assert p.returncode == 0, o[-3000:]
        res.append(json.loads(next(ln for ln in o.splitlines() if ln.startswith("RESULT "))[7:]))
    assert all(r["max_param_diff_to_rank0"] == 0.0 for r in res), res
    assert all(r["grad_left"] == 0.0 for r in res)
    assert res[0]["losses"] != res[1]["losses"]                   # different data ...
    assert all(r["losses"][-1] < r["losses"][0] for r in res)     # ... both learning


WORKER_SCRIPT = """
import os, sys, json
sys.path.insert(0, {root!r}); sys.path.insert(0, os.path.join({root!r}, "tests"))
import kernel_emulation as ke
ke.install()
from trainingjob_operator_b200.runtime import worker as W
W.build_adapter = lambda args, device: W.EngineAdapter(args.model, args.batch, args.seq, args, device="cpu")
sys.exit(W.main(sys.argv[1:]))
"""


def run_workers(tmp_path, n, argv, env_extra=None, timeout=600):
    """The real worker entry point (``runtime/worker.py main``) with the engine adapter on CPU: n gloo ranks."""
    import json
    import socket

    script = tmp_path / "worker_cpu.py"
    script.write_text(textwrap.dedent(WORKER_SCRIPT.format(root=ROOT)))
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    procs = []
    for r in range(n):
        env = dict(os.environ, RANK=str(r), WORLD_SIZE=str(n), LOCAL_RANK=str(r), MASTER_ADDR="127.0.0.1",
                   MASTER_PORT=str(port), OMP_NUM_THREADS="2", AITJ_WORKDIR=str(tmp_path), TRAININGJOB_NAME="dry",
                   **(env_extra or {}))
        env.pop("AITJ_MASTER", None)
        res = tmp_path / f"result{r}.json"
        procs.append((res, subprocess.Popen([sys.executable, str(script), "--cpu", "--result", str(res)] + argv, env=env,
                                            stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    out = []
    for res, p in procs:
        log = p.communicate(timeout=timeout)[0]
        assert p.returncode == 0, log[-4000:]
        out.append((json.load(open(res)) if res.exists() else None, log))
    return out


@pytest.mark.slow
def test_worker_loop_with_the_engine_adapter_single_rank_checkpoint_and_resume(tmp_path):
    """``worker.run`` end to end on one rank: warm-up, timed region, checkpoints every 2 steps, result record; then the
    same job restarted (TRAININGJOB_REPLICA_RESTARTCOUNT=1) resumes from the checkpoint past the warm-up and still
    produces a throughput record."""
    argv = ["--model", "gpt2-tiny", "--batch", "2", "--seq", "128", "--steps", "4", "--warmup", "3", "--ckpt-every", "2",
            "--ckpt-dir", str(tmp_path / "ck")]
    (r, log), = run_workers(tmp_path, 1, argv, {"AITJ_CKPT_ASYNC": "0"})
    assert r and r["steps_done"] == 7 and r["world"] == 1 and r["samples_per_sec"] > 0, (r, log[-2000:])
    assert r["loss_last"] < r["loss_first"]
    (r2, log2), = run_workers(tmp_path, 1, argv, {"AITJ_CKPT_ASYNC": "0", "TRAININGJOB_REPLICA_RESTARTCOUNT": "1"})
    assert "resumed from checkpoint at step 6" in log2, log2[-2000:]
    assert r2 and r2["steps_done"] == 7 and r2["samples_per_sec"] > 0


@pytest.mark.slow
def test_worker_loop_with_the_engine_adapter_two_ranks(tmp_path):
    """Two gloo ranks through rendezvous, the elected state hand-off (flat engine state), bucketed gradient sync and the
    max-over-ranks timing: both ranks report the same loss trajectory end point and world size 2."""
    argv = ["--model", "bert-tiny", "--batch", "2", "--seq", "128", "--steps", "3", "--warmup", "3"]
    res = run_workers(tmp_path, 2, argv)
    r0 = res[0][0]
    assert r0 and r0["world"] == 2 and r0["global_batch"] == 4 and r0["steps_done"] == 6, (r0, res[0][1][-2000:])
    assert "gradient sync" in res[0][1]


@pytest.mark.slow
def test_engine_worker_through_the_control_plane_elastic_rescale_and_in_place_recovery(tmp_path):
    """The engine adapter (emulated kernels, CPU / gloo) as the workers of a ``faultTolerant`` elastic job submitted
    through ``LocalCluster``: scale 1 -> 2 hands the flat engine state (fp32 master weights + moments) to the joiner and
    re-binds the trainer; SIGKILL of rank 1 is repaired in place -- the survivor keeps its process, the replacement
    receives the state again.  On GPUs this is the path of tools/elastic_gpu_check.py / fault_check.py --fault-tolerant."""
    import json
    import signal
    import time

    from trainingjob_operator_b200.api import constants as C
    from trainingjob_operator_b200.cmd.local import LocalCluster
    from trainingjob_operator_b200.cmd.options import TrainingJobOperatorOption

    script = tmp_path / "worker_cpu.py"
    script.write_text(textwrap.dedent(WORKER_SCRIPT.format(root=ROOT)))
    worker = [sys.executable, str(script), "--cpu", "--model", "gpt2-tiny", "--batch", "2", "--seq", "128", "--steps", "0",
              "--elastic", "--ckpt-every", "0", "--step-sleep", "0.05"]
    job = {"apiVersion": C.API_VERSION, "kind": C.KIND, "metadata": {"name": "eng"},
           "spec": {"frameworkType": "pytorch", "faultTolerant": True, "replicaSpecs": {"trainer": {
               "replicas": 1, "minReplicas": 1, "maxReplicas": 2, "edlPolicy": "Manual", "restartPolicy": "OnFailure",
               "restartLimit": 4,
               "template": {"spec": {"terminationGracePeriodSeconds": 1, "containers": [{
                   "name": "aitj-trainer", "command": worker, "workingDir": ROOT,
                   "env": [{"name": "PYTHONPATH", "value": ROOT}, {"name": "OMP_NUM_THREADS", "value": "2"}]}]}}}}}}

    def wait(fn, timeout=120.0):
        t0 = time.time()
        while time.time() - t0 < timeout:
            try:
                v = fn()
                if v:
                    return v
            except Exception:  # noqa: BLE001
                pass
            time.sleep(0.05)
        raise TimeoutError

    def trace(lc, key):
        return json.loads(lc.jobs().get("eng").annotations.get(f"aitj.b200/{key}", "null"))

    def pids(lc):
        return {sid.split("/")[1]: p for sid, p in lc.agent.sup.list() if "/eng-trainer-" in sid}

    with LocalCluster(num_gpus=0, workdir=str(tmp_path / "wd"), option=TrainingJobOperatorOption(thread_num=2)) as lc:
        try:
            lc.apply(job)
            wait(lambda: (trace(lc, "worker-trace") or {}).get("first_step_done"))
            p0 = pids(lc)["eng-trainer-0"]
            lc.jobs().patch("eng", {"spec": {"replicaSpecs": {"trainer": {"replicas": 2}}}})
            rec = wait(lambda: (lambda r: r if r and r.get("world") == 2 else None)(trace(lc, "rescale-trace")))
            assert rec["generation"] == 2 and pids(lc)["eng-trainer-0"] == p0
            log1 = open(os.path.join(lc.workdir, "logs", "default_eng-trainer-1_aitj-trainer.log")).read()
            assert "joined generation 2 (world 2) at step" in log1
            # ---- SIGKILL rank 1: in-place recovery
            os.kill(pids(lc)["eng-trainer-1"], signal.SIGKILL)
            rec = wait(lambda: (lambda r: r if r and r.get("generation", 0) >= 3 and r.get("recovered_from") else None)(
                trace(lc, "rescale-trace")))
            assert rec["world"] == 2
            j = wait(lambda: (lambda x: x if x.status.phase == "Running" and
                              x.status.replica_statuses["trainer"].active == 2 else None)(lc.jobs().get("eng")))
            assert j.status.restart_counts == {"trainer": 1}
            assert pids(lc)["eng-trainer-0"] == p0                       # the survivor was never restarted
            log0 = open(os.path.join(lc.workdir, "logs", "default_eng-trainer-0_aitj-trainer.log")).read()
            assert "lost a peer" in log0 and "keeping state" in log0
            # ---- scale back down: rank 1 leaves, rank 0 trains on alone
            lc.jobs().patch("eng", {"spec": {"replicaSpecs": {"trainer": {"replicas": 1}}}})
            rec = wait(lambda: (lambda r: r if r and r.get("world") == 1 else None)(trace(lc, "rescale-trace")))
            assert pids(lc)["eng-trainer-0"] == p0
        finally:
            lc.jobs().delete("eng")
            time.sleep(0.5)


HANG_WORKER_SCRIPT = """
import os, sys, threading, time
sys.path.insert(0, {root!r})
import torch.distributed as dist
from trainingjob_operator_b200.runtime import worker as W, rendezvous as R

# NCCL semantics on gloo: a collective whose peer died does not raise -- it never completes -- until the communicator is
# aborted, after which it fails.  (gloo raises after the group's short time-out; that error is turned into the hang.)
ABORT = threading.Event()

def nccl_like(fn):
    def w(*a, **k):
        try:
            return fn(*a, **k)
        except RuntimeError as e:
            t0 = time.time()
            print(f"[emulation] collective failed ({{type(e).__name__}}): hanging like NCCL until the communicator is aborted", flush=True)
            while not ABORT.is_set():
                if time.time() - t0 > 90:
                    print("[emulation] nobody aborted the communicator: this rank would hang for ever", flush=True)
                    os._exit(99)
                time.sleep(0.02)
            raise RuntimeError("NCCL communicator was aborted") from None
    return w

_teardown = R.teardown_group
def teardown(broken=False):
    if broken:
        ABORT.set()
    _teardown(broken)
R.teardown_group = W.teardown_group = teardown
_init = R.init_process_group
def init(*a, **k):
    out = _init(*a, **k)
    ABORT.clear()
    return out
R.init_process_group = init
dist.all_reduce = nccl_like(dist.all_reduce)
dist.broadcast = nccl_like(dist.broadcast)
_build = W.build_adapter
def build(args, device):
    ad = _build(args, device)
    ad.train_step = nccl_like(ad.train_step)
    return ad
W.build_adapter = build
sys.exit(W.main(sys.argv[1:]))
"""


@pytest.mark.slow
@pytest.mark.parametrize("model", ["mlp", "bert-tiny"])
def test_stall_breaker_recovers_four_ranks_whose_collectives_hang_like_nccl(tmp_path, model):
    """(``bert-tiny``: the engine adapter with emulated kernels -- the flat engine state is what is handed over.)
    BASELINE config 4's shape (4 ranks, SIGKILL rank 3, ``faultTolerant``) with collectives that HANG when a peer dies,
    as NCCL's do, instead of raising as gloo's do: every survivor sits inside its step (or inside the generation
    agreement) until its StallBreaker -- armed with AITJ_STALL_BREAKER=force -- sees the newer generation and aborts the
    communicator; then all three re-rendezvous with the replacement and go on, processes kept.  A second victim (rank 0,
    the state source) is killed afterwards.  This is the logic that could not be diagnosed on 4 GPUs in round 2."""
    import json
    import signal
    import time

    from trainingjob_operator_b200.api import constants as C
    from trainingjob_operator_b200.cmd.local import LocalCluster
    from trainingjob_operator_b200.cmd.options import TrainingJobOperatorOption

    script = tmp_path / "hang_worker.py"
    src = HANG_WORKER_SCRIPT.format(root=ROOT)
    shape = ["--model", "mlp", "--batch", "16"]
    if model != "mlp":
        src = src.replace("_build = W.build_adapter", "sys.path.insert(0, os.path.join({root!r}, 'tests'))\n"
                          "import kernel_emulation as ke\nke.install()\n"
                          "_build = lambda args, device: W.EngineAdapter(args.model, args.batch, args.seq, args, device='cpu')"
                          .format(root=ROOT))
        shape = ["--model", model, "--batch", "2", "--seq", "128"]
    script.write_text(textwrap.dedent(src))
    worker = [sys.executable, str(script), "--cpu"] + shape + ["--steps", "0", "--elastic", "--ckpt-every", "10",
                                                                "--step-sleep", "0.05"]
    env = [{"name": "PYTHONPATH", "value": ROOT}, {"name": "OMP_NUM_THREADS", "value": "1"},
           {"name": "AITJ_STALL_BREAKER", "value": "force"}, {"name": "AITJ_FT_ABORT_AFTER", "value": "1.5"},
           {"name": "AITJ_COLLECTIVE_TIMEOUT", "value": "2"}]
    job = {"apiVersion": C.API_VERSION, "kind": C.KIND, "metadata": {"name": "hang"},
           "spec": {"frameworkType": "pytorch", "faultTolerant": True, "replicaSpecs": {"trainer": {
               "replicas": 4, "minReplicas": 4, "maxReplicas": 4, "edlPolicy": "Manual", "restartPolicy": "OnFailure",
               "restartLimit": 6,
               "template": {"spec": {"terminationGracePeriodSeconds": 1, "containers": [{
                   "name": "aitj-trainer", "command": worker, "workingDir": ROOT, "env": env}]}}}}}}

    def wait(fn, timeout=150.0):
        t0 = time.time()
        while time.time() - t0 < timeout:
            try:
                v = fn()
                if v:
                    return v
            except Exception:  # noqa: BLE001
                pass
            time.sleep(0.05)
        raise TimeoutError

    def ann(lc, key):
        return json.loads(lc.jobs().get("hang").annotations.get(f"aitj.b200/{key}", "null"))

    def pids(lc):
        return {sid.split("/")[1]: p for sid, p in lc.agent.sup.list() if "/hang-trainer-" in sid}

    def logs(lc, i):
        return open(os.path.join(lc.workdir, "logs", f"default_hang-trainer-{i}_aitj-trainer.log")).read()

    with LocalCluster(num_gpus=0, workdir=str(tmp_path / "wd"), option=TrainingJobOperatorOption(thread_num=2)) as lc:
        try:
            lc.apply(job)
            wait(lambda: (ann(lc, "worker-trace") or {}).get("first_step_done"))
            time.sleep(1.0)
            before = pids(lc)
            os.kill(before["hang-trainer-3"], signal.SIGKILL)
            rec = wait(lambda: (lambda r: r if r and r.get("generation", 0) >= 2 and r.get("recovered_from") else None)(
                ann(lc, "rescale-trace")))
            assert rec["world"] == 4
            wait(lambda: (lambda x: x.status.phase == "Running" and
                          x.status.replica_statuses["trainer"].active == 4)(lc.jobs().get("hang")))
            now = pids(lc)
            assert all(now[k] == before[k] for k in ("hang-trainer-0", "hang-trainer-1", "hang-trainer-2")), (before, now)
            tripped = [i for i in range(3) if "aborting the communicator" in logs(lc, i)]
            assert tripped, "no survivor's breaker fired: the recovery did not go through the NCCL-like path"
            assert all("hanging like NCCL" in logs(lc, i) for i in range(3))
            assert lc.jobs().get("hang").status.restart_counts == {"trainer": 1}
            # ---- second victim: rank 0 (the rank the others take their state from)
            gen = ann(lc, "rescale-trace")["generation"]
            before = pids(lc)
            t_kill = time.time()
            os.kill(before["hang-trainer-0"], signal.SIGKILL)
            rec = wait(lambda: (lambda r: r if r and r.get("generation", 0) > gen and r.get("recovered_from") else None)(
                ann(lc, "rescale-trace")))
            # the survivors' trainers were warm: the breaker's ordinary threshold applies (not the 30 s it grants the
            # first step after a re-bind), also when the rank sits in the generation agreement rather than in the step
            assert rec["at"] - t_kill < 15.0, rec["at"] - t_kill
            wait(lambda: (lambda x: x.status.phase == "Running" and
                          x.status.replica_statuses["trainer"].active == 4)(lc.jobs().get("hang")))
            now = pids(lc)
            assert all(now[k] == before[k] for k in ("hang-trainer-1", "hang-trainer-2", "hang-trainer-3"))
            assert lc.jobs().get("hang").status.restart_counts == {"trainer": 2}
        finally:
            for i in range(4):
                try:
                    sys.stderr.write(f"---- rank {i}\\n" + logs(lc, i)[-1500:] + "\\n")
                except Exception:  # noqa: BLE001
                    pass
            lc.jobs().delete("hang")
            time.sleep(0.5)


@pytest.mark.slow
def test_stall_exit_makes_a_pod_scope_restart_whole_again_in_seconds(tmp_path):
    """``restartScope: Pod`` without ``faultTolerant``: the controller re-creates only the killed replica; the survivor
    sits in a collective that (NCCL-like) never returns.  Round 1 measured 32.7 s for this on GPUs because the survivor
    was only removed by the agent's 20 s heartbeat time-out.  The worker's stall-exit breaker leaves with 137 as soon as
    the controller's repair (a newer rendezvous generation) is visible, the controller replaces it too, and both
    replicas resume from the checkpoint."""
    import json
    import signal
    import time

    from trainingjob_operator_b200.api import constants as C
    from trainingjob_operator_b200.cmd.local import LocalCluster
    from trainingjob_operator_b200.cmd.options import TrainingJobOperatorOption

    script = tmp_path / "hang_worker.py"
    script.write_text(textwrap.dedent(HANG_WORKER_SCRIPT.format(root=ROOT)))
    worker = [sys.executable, str(script), "--cpu", "--model", "mlp", "--batch", "16", "--steps", "0", "--ckpt-every", "5",
              "--step-sleep", "0.05"]
    env = [{"name": "PYTHONPATH", "value": ROOT}, {"name": "OMP_NUM_THREADS", "value": "1"},
           {"name": "AITJ_STALL_BREAKER", "value": "force"}, {"name": "AITJ_STALL_EXIT_AFTER", "value": "1.5"},
           {"name": "AITJ_COLLECTIVE_TIMEOUT", "value": "1"}, {"name": "AITJ_HANG_TIMEOUT", "value": "60"}]
    job = {"apiVersion": C.API_VERSION, "kind": C.KIND, "metadata": {"name": "podscope"},
           "spec": {"frameworkType": "pytorch", "replicaSpecs": {"trainer": {
               "replicas": 2, "restartPolicy": "OnFailure", "restartScope": "Pod", "restartLimit": 6,
               "template": {"spec": {"terminationGracePeriodSeconds": 1, "containers": [{
                   "name": "aitj-trainer", "command": worker, "workingDir": ROOT, "env": env}]}}}}}}

    def wait(fn, timeout=120.0):
        t0 = time.time()
        while time.time() - t0 < timeout:
            try:
                v = fn()
                if v:
                    return v
            except Exception:  # noqa: BLE001
                pass
            time.sleep(0.05)
        raise TimeoutError

    def first_step(lc):
        return (json.loads(lc.jobs().get("podscope").annotations.get("aitj.b200/worker-trace", "null")) or {}).get(
            "first_step_done", 0.0)

    with LocalCluster(num_gpus=0, workdir=str(tmp_path / "wd"), option=TrainingJobOperatorOption(thread_num=2)) as lc:
        try:
            lc.apply(job)
            wait(lambda: first_step(lc) > 0)
            time.sleep(1.5)                                            # a checkpoint exists
            pid = next(p for sid, p in lc.agent.sup.list() if "/podscope-trainer-1/" in sid)
            t_kill = time.time()
            os.kill(pid, signal.SIGKILL)
            wait(lambda: first_step(lc) > t_kill)
            took = first_step(lc) - t_kill
            j = lc.jobs().get("podscope")
            assert j.status.restart_counts == {"trainer": 2}, j.status.restart_counts     # the victim and the survivor
            log0 = open(os.path.join(lc.workdir, "logs", "default_podscope-trainer-0_aitj-trainer.log")).read()
            assert "does not recover in place" in log0 and "leaving (137)" in log0
            assert "resumed from checkpoint" in log0
            assert took < 15.0, took            # seconds, not the 60 s heartbeat time-out configured above
        finally:
            lc.jobs().delete("podscope")
            time.sleep(0.5)


def test_owner_sharded_data_parallel_equals_one_replica_on_the_joint_batch(monkeypatch, tmp_path):
    """The default multi-GPU algorithm (``AITJ_ALLREDUCE=rs``) with its peer-memory kernels emulated: two "ranks" (threads
    with a real barrier where the device-side barriers are) each see half of a batch; gradient producers add every
    piece into the copy of the rank that OWNS it, the owner clips on the exchanged partial norms and runs AdamW on its
    shard only, and the bf16 parameters are stored into every rank's copy.  After three steps: (a) nothing is left in
    any gradient buffer, (b) every rank holds the same bf16 parameters, (c) they equal -- to rounding -- those of ONE
    engine that trained on the joint batch, as do the fp32 master weights of each rank's own shard."""
    import threading

    from trainingjob_operator_b200.models.gpt2 import GPT2Config, GPT2Engine

    ke.install(monkeypatch)
    cfg = GPT2Config(vocab_size=1000, n_layer=2, n_head=4, n_embd=256, block_size=128, name="t")
    B, T, N, STEPS = 2, 128, 2, 3
    g = torch.Generator().manual_seed(11)
    toks = [torch.randint(0, cfg.vocab_size, (N * B, T), generator=g) for _ in range(STEPS)]

    def perturb(eng):
        gg = torch.Generator().manual_seed(9)
        for s_ in eng.params.specs:
            if len(s_.shape) == 1:
                eng.params.w32(s_.name).add_(torch.randn(s_.shape, generator=gg) * 0.05)
        eng.params.refresh_compute_copy()

    # ---- reference: one replica, the joint batch
    ref = GPT2Engine(cfg, N * B, T, "cpu", seed=3, gemm_backend="wgmma")
    perturb(ref)
    for step in range(STEPS):
        ref.tok.copy_(toks[step].view(-1))
        ref.tgt.copy_(torch.roll(toks[step], -1, dims=1).reshape(-1))
        ref.forward()
        ref.backward()
        ref.optimizer_step(lr=1e-3, step=step + 1, max_norm=0.5)

    # ---- two owner-sharded ranks
    fw = ke.FakeWorld(N)
    ke._CURRENT["world"] = fw
    engs = []
    for r in range(N):
        e = GPT2Engine(cfg, B, T, "cpu", seed=3, gemm_backend="wgmma")
        perturb(e)
        fw.attach(e.params)
        engs.append(e)
    sh0 = fw.shards[0]
    assert sh0.bounds[0] == 0 and sh0.bounds[-1] == engs[0].params.total and 0 < sh0.bounds[1] < sh0.bounds[2]
    errors = []

    def rank_main(r):
        try:
            e, sh = engs[r], fw.shards[r]
            for step in range(STEPS):
                mine = toks[step][r * B:(r + 1) * B]
                e.tok.copy_(mine.reshape(-1))
                e.tgt.copy_(torch.roll(mine, -1, dims=1).reshape(-1))
                e.forward()
                e.backward()
                sh.barrier()                       # runtime/trainer.py:_device_step: every contribution has landed
                e.optimizer_step(lr=1e-3, step=step + 1, max_norm=0.5, grad_div=float(N))
                sh.barrier()                       # every rank's bf16 parameters arrived, every shard is zeroed
        except Exception as ex:  # noqa: BLE001
            errors.append((r, repr(ex)))
            fw.sync.abort()

    threads = [threading.Thread(target=rank_main, args=(r,)) for r in range(N)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(300)
    assert not errors, errors
    total = engs[0].params.total
    for r, e in enumerate(engs):
        sh = fw.shards[r]
        assert sh.barriers == 3 * STEPS                                      # three device barriers per step
        assert float(sh.g[:total].abs().max()) == 0.0                        # (a) owned range zeroed by the sweep,
        assert float(e.params.g_small.abs().max()) == 0.0                    #     nothing left behind elsewhere
        assert torch.equal(e.params.p16, engs[0].params.p16)                 # (b)
        own = slice(sh.lo, sh.hi)
        assert rel(e.params.p32[own], ref.params.p32[own]) < 2e-4, r         # (c) fp32 master weights of the shard
    assert rel(engs[0].params.p16.float(), ref.params.p16.float()) < 2e-3    # (c) all-gathered bf16 copy
    # the clip really engaged (max_norm 0.5 is below the gradient norm of this model), from the exchanged partial norms
    assert float(fw.shards[0].parts[:N].sum()) > 0.25
    # ... and with the right scale: the ranks' shards hold the SUM over ranks of per-rank mean gradients, the sweep divides
    # by the world size, so sqrt(sum of partial square sums) / N is the joint batch's gradient norm (Adam's update is
    # scale-invariant, so this is the assertion that sees a wrong grad_div or a double-counted contribution)
    joint = float(ref.sumsq) ** 0.5
    sharded = float(fw.shards[1].parts[:N].sum()) ** 0.5 / N
    assert abs(sharded - joint) < 2e-3 * joint, (sharded, joint)
    # bench.py --dump-outputs: every rank gathers the shards (EngineAdapter.prepare_state, a collective -- broadcasts
    # emulated between the two threads), then rank 0 writes its fp32 master weights: they must be the joint-batch
    # replica's everywhere, not only in rank 0's own shard
    from trainingjob_operator_b200.runtime import worker as W

    assert rel(engs[0].params.p32, ref.params.p32) > 1e-2               # before the gather: rank 1's shard is stale
    sync = threading.Barrier(N)
    box, me = {}, threading.local()

    def fake_broadcast(t, src):
        me.calls = getattr(me, "calls", 0) + 1
        if me.rank == src:
            box[me.calls] = t.clone()
        sync.wait()
        if me.rank != src:
            t.copy_(box[me.calls])
        sync.wait()

    real = (W.dist.is_initialized, W.dist.broadcast)
    monkeypatch.setattr(W.dist, "is_initialized", lambda: True)
    monkeypatch.setattr(W.dist, "broadcast", fake_broadcast)
    adapters = [types.SimpleNamespace(engine=e, state_tensors=e.params.state_tensors) for e in engs]

    def gather(r):
        me.rank = r
        W.EngineAdapter.prepare_state(adapters[r])

    threads = [threading.Thread(target=gather, args=(r,)) for r in range(N)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(120)
    W.dump_outputs(str(tmp_path), adapters[0], [1.0, 2.0])
    dumped = torch.from_numpy(np.load(tmp_path / "weights_sample.npy"))
    assert dumped.numel() == ref.params.p32.numel()
    assert rel(dumped, ref.params.p32) < 2e-4
    assert np.load(tmp_path / "losses.npy").tolist() == [1.0, 2.0]
    monkeypatch.setattr(W.dist, "is_initialized", real[0])
    monkeypatch.setattr(W.dist, "broadcast", real[1])
    # leaving the sharded mode (world shrank to one rank, re-bind after a re-rendezvous): private buffers again, the bf16
    # parameters kept, gradients plain local tensors
    P = engs[0].params
    kept = P.p16.clone()
    P.detach_shard()
    assert P.shard is None and P.g_small is None and torch.equal(P.p16, kept) and P.p16 is not fw.shards[0].w
    assert isinstance(P.grad("h0.fc_w"), torch.Tensor) and float(P.g32.abs().max()) == 0.0


def test_bert_layout_can_be_owner_sharded(monkeypatch):
    """The owner-sharded mode needs every 1-D parameter in one tail region of the flat layout and 32-row / 256-element
    aligned ownership bounds: BERT's layout (three embedding tables, MLM head, decoder bias) qualifies, for 2..8 ranks."""
    from trainingjob_operator_b200.models.bert import BertConfig, BertEngine
    from trainingjob_operator_b200.parallel.symm import shard_bounds

    ke.install(monkeypatch)
    eng = BertEngine(BertConfig.tiny(), 2, 128, "cpu", seed=3)
    P = eng.params
    for world in (2, 3, 4, 8):
        b = shard_bounds(P.specs, P.total, world)
        assert len(b) == world + 1 and b[0] == 0 and b[-1] == P.total and all(x % 256 == 0 for x in b)
        assert all(b[i] <= b[i + 1] for i in range(world))
        for x in b[1:-1]:                      # a bound inside a 2-D tensor sits on a multiple of 32 rows
            s_ = next(s for s in P.specs if s.offset <= x < s.offset + s.padded)
            if len(s_.shape) == 2 and x < s_.offset + s_.numel:
                assert (x - s_.offset) % (32 * s_.shape[1]) == 0, (world, s_.name)
    fw = ke.FakeWorld(2)
    fw.attach(P)
    lo, hi = P.small_range
    assert all((len(s_.shape) == 1) == (lo <= s_.offset < hi) for s_ in P.specs)


@pytest.mark.parametrize("model", ["gpt2", "bert"])
@pytest.mark.parametrize("segment_join", [False, True], ids=["one-graph", "segments"])
def test_side_stream_weight_gradients_have_no_ordering_hazard(monkeypatch, model, segment_join):
    """``AITJ_WGRAD_STREAM=1`` launches the weight-gradient GEMMs on a side stream.  Here that stream runs everything as
    LATE as its events allow (``kernel_emulation.LateStream``): if the main stream could overwrite an operand of a pending
    weight-gradient GEMM, or read a gradient before it exists, the result differs from the reference model.  Checked for
    both engines, in the one-graph mode and with a join at the end of every backward segment (bucketed DDP)."""
    ke.install(monkeypatch)
    if model == "gpt2":
        cfg, eng, ref, tok, tgt = gpt2_pair(monkeypatch)
        names, ref_loss = GPT2_GRADS, (lambda: ref(tok, tgt))
    else:
        from trainingjob_operator_b200.models.bert import BertConfig, BertEngine, BertReference, SyntheticMLM

        cfg = BertConfig.tiny()
        B, T = 2, 128
        eng = BertEngine(cfg, B, T, "cpu", seed=3)
        g = torch.Generator().manual_seed(9)
        for s_ in eng.params.specs:
            if len(s_.shape) == 1:
                eng.params.w32(s_.name).add_(torch.randn(s_.shape, generator=g) * 0.05)
        eng.params.w32("dec_b")[cfg.vocab_size:].zero_()
        eng.params.refresh_compute_copy()
        ref = BertReference(cfg, eng.params)
        tok, typ, lab = SyntheticMLM(cfg.vocab_size, B, T, n_batches=1, seed=5, pin=False).next()
        for dst, src in zip(eng.input_tensors(), (tok, typ, lab)):
            dst.copy_(src)
        names = ("wte", "wpe", "wtt", "h0.qkv_w", "h0.proj_w", "h0.fc_w", "h0.fc2_w", "h1.qkv_w", "h1.proj_w", "h1.fc_w",
                 "h1.fc2_w", "mlm_w", "h0.fc_b", "h1.ln2_b")
        ref_loss = lambda: ref(tok.view(B, T), typ.view(B, T), lab.view(B, T))          # noqa: E731
    ke.install_late_streams(monkeypatch)          # (after the engines exist: wraps the emulated kernels installed above)
    side = ke.LateStream()
    eng.wgrad_stream = side
    eng.segment_join = segment_join
    eng.params.g32.zero_()
    eng.forward()
    eng.backward()
    assert side.done == len(side.queue) > 0, "weight-gradient GEMMs left unexecuted: a join is missing"
    if not segment_join:
        assert side.reordered > 0           # the model really ran them behind later main-stream work
    loss = ref_loss()
    loss.backward()
    for name in names:
        gref, got = ref.p(name).grad, eng.params.grad(name)
        assert rel(got, gref) < 6e-2, (name, rel(got, gref))


@pytest.mark.parametrize("model", ["gpt2", "bert"])
@pytest.mark.parametrize("side_stream", [False, True], ids=["in-line", "side-stream"])
def test_gradient_buckets_are_final_when_their_hook_fires(monkeypatch, model, side_stream):
    """Bucketed DDP starts a bucket's all-reduce the moment the engine calls ``grad_hook(bucket)``: from then on nothing may
    add to that slice of the flat gradient buffer (the tied embedding gets contributions from the head AND the tail; the
    1-D parameters from every layer).  The hook here snapshots the slice; at the end of backward it must be unchanged --
    also with the weight-gradient GEMMs on the late-running side stream, where the per-segment join is what guarantees it."""
    ke.install(monkeypatch)
    if model == "gpt2":
        cfg, eng, ref, tok, tgt = gpt2_pair(monkeypatch)
    else:
        from trainingjob_operator_b200.models.bert import BertConfig, BertEngine, SyntheticMLM

        cfg = BertConfig.tiny()
        eng = BertEngine(cfg, 2, 128, "cpu", seed=3)
        for dst, src in zip(eng.input_tensors(), SyntheticMLM(cfg.vocab_size, 2, 128, n_batches=1, seed=5, pin=False).next()):
            dst.copy_(src)
    if side_stream:
        ke.install_late_streams(monkeypatch)
        eng.wgrad_stream = ke.LateStream()
    eng.segment_join = True                       # what EngineTrainer sets when a bucket reducer is attached
    ranges = {name: (a, b) for name, a, b in eng.grad_buckets()}
    assert sum(b - a for a, b in ranges.values()) == eng.params.total          # the buckets tile the whole buffer
    seen = {}

    def hook(name):
        assert name in ranges and name not in seen, name
        a, b = ranges[name]
        seen[name] = eng.params.g32[a:b].clone()

    eng.grad_hook = hook
    eng.params.g32.zero_()
    eng.forward()
    eng.backward()
    assert set(seen) == set(ranges)
    for name, snap in seen.items():
        a, b = ranges[name]
        assert torch.equal(snap, eng.params.g32[a:b]), f"bucket {name} was still written after its hook"
        assert float(snap.abs().max()) > 0
