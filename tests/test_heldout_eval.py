"""Held-out evaluation of GPT-2 workers (``--eval-data``): the cross-entropy epilogue of the logits GEMM (``EPI_XENT``,
``gemm_xent`` + ``xent_finish``), ``GPT2Engine.eval_forward``, the worker's sample assignment, schedule and reports.

CPU tests run the engine with the kernel entry points emulated (``tests/kernel_emulation.py``, whose ``gemm_xent`` /
``xent_finish`` keep the kernels' partial layout) and gloo between processes; the GPU tests run the
hand-written kernels on an H100."""
import io
import json
import os
import re
import socket
import subprocess
import sys
import textwrap
import types

import numpy as np
import pytest
import torch

import kernel_emulation as ke
from test_gemm_epilogue_variants import _compiled_pairs, variants  # noqa: F401  (module fixture)
from test_gemm_sass import gemm_sass  # noqa: F401  (module fixture: name -> SASS lines of every GEMM instantiation)
from test_packed_documents import install_doc_attention, structured_corpus, write_llmc
from trainingjob_operator_b200.ops import functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTS = os.path.dirname(os.path.abspath(__file__))


# ------------------------------------------------------------------------------------ emulated entry points
XENT_CALLS = ke.XENT_CALLS
gemm_xent, xent_finish = ke.gemm_xent, ke.xent_finish


def install_xent(monkeypatch=None):
    """The cross-entropy entry points alone (``kernel_emulation.install`` includes them)."""
    for name, fn in (("gemm_xent", gemm_xent), ("xent_finish", xent_finish)):
        if monkeypatch is not None:
            monkeypatch.setattr(F, name, fn)
        else:
            setattr(F, name, fn)


def _cfg():
    from trainingjob_operator_b200.models.gpt2 import GPT2Config

    return GPT2Config(vocab_size=1000, n_layer=2, n_head=4, n_embd=256, block_size=128, name="t")


def _args(**kw):
    from trainingjob_operator_b200.runtime.worker import parse_args

    argv = ["--model", "gpt2-tiny", "--seq", "128"]
    for k, v in kw.items():
        argv += [f"--{k.replace('_', '-')}", str(v)]
    return parse_args(argv)


# ------------------------------------------------------------------------------------ the emulation itself
def test_emulated_partials_give_the_log_softmax_loss():
    g = torch.Generator().manual_seed(0)
    x = torch.randn(300, 64, generator=g).bfloat16()
    w = (torch.randn(520, 64, generator=g) * 4).bfloat16()
    V = 389                                  # blocks 3 and 4 hold no vocabulary column
    target = torch.randint(0, V, (300,), generator=g)
    target[::9] = -1
    part = torch.zeros(300, F.xent_blocks(520), 2)
    t, loss, acc = torch.zeros(300), torch.zeros(300), torch.zeros(2, dtype=torch.float64)
    gemm_xent(x, w, target, V, part, t, block_n=512)
    xent_finish(part, t, target, loss, acc)
    z = (x.double() @ w.double().t())[:, :V]
    ref = torch.logsumexp(z, 1) - z.gather(1, target.clamp(min=0)[:, None])[:, 0]
    ref = torch.where(target >= 0, ref, torch.zeros_like(ref))
    assert float((loss.double() - ref).abs().max()) < 1e-4
    assert float(acc[1]) == int((target >= 0).sum()) and abs(float(acc[0]) - float(ref.sum())) < 1e-2


# ------------------------------------------------------------------------------------ 1. sample assignment
@pytest.mark.parametrize("W", [1, 2, 3, 5])
def test_every_held_out_window_is_evaluated_once_at_any_world_size(monkeypatch, tmp_path, W):
    """S = 27 windows in micro-batches of B = 4: seven micro-batches, the last with three rows of padding."""
    ke.install(monkeypatch)
    install_xent(monkeypatch)
    from trainingjob_operator_b200.runtime.worker import EngineAdapter

    shard = write_llmc(tmp_path / "val_000.bin", structured_corpus(20000, 1000, 999, 1))
    B, S = 4, 27
    a = EngineAdapter("gpt2-tiny", B, 128, _args(batch=B, eval_data=shard, eval_samples=S), device="cpu")
    seen = []
    for r in range(W):
        a.trainer = types.SimpleNamespace(world=W, rank=r)
        assert a.eval_plan().micro == tuple(range(r, 7, W))
        for tok, tgt in a._eval_inputs():
            rows = a.eval_data.samples_read
            seen += rows
            t = tgt.view(B, 128)
            assert bool((t[:len(rows)] >= 0).all()), "a window of the held-out set carries a padding target"
            assert bool((t[len(rows):] == -1).all()) and bool((tok.view(B, 128)[len(rows):] == 0).all())
    assert sorted(seen) == list(range(S))


# ------------------------------------------------------------------------------------ 2. engine against the reference
def _eval_engine(monkeypatch, doc_mask):
    from trainingjob_operator_b200.models.gpt2 import GPT2Engine, GPT2Reference

    (install_doc_attention if doc_mask else ke.install)(monkeypatch)
    install_xent(monkeypatch)
    cfg = _cfg()
    B, T = 2, 128
    eng = GPT2Engine(cfg, B, T, "cpu", seed=3, doc_mask=doc_mask)
    g = torch.Generator().manual_seed(5)
    tok = torch.randint(0, cfg.vocab_size - 1, (B, T), generator=g)
    tok[0, 40] = tok[1, 77] = 999
    tgt = torch.roll(tok, -1, dims=1)
    tgt[1, 100:] = -1                        # padding rows
    ins = [tok, tgt]
    if doc_mask:
        from trainingjob_operator_b200.runtime.data import doc_starts

        ins.append(torch.from_numpy(doc_starts(tok.numpy(), 999)))
    for dst, src in zip(eng.input_tensors(), ins):
        dst.copy_(src.reshape(-1))
    return eng, GPT2Reference(cfg, eng.params), ins


@pytest.mark.parametrize("doc_mask", [False, True])
def test_eval_forward_matches_the_reference_and_leaves_the_state_alone(monkeypatch, doc_mask):
    eng, ref, ins = _eval_engine(monkeypatch, doc_mask)
    P = eng.params
    P.g32.normal_(generator=torch.Generator().manual_seed(1))
    P.m.normal_(generator=torch.Generator().manual_seed(2))
    eng.logits.fill_(0.5)
    before = [t.clone() for t in (P.p32, P.m, P.v, P.g32, P.p16, eng.logits)]
    XENT_CALLS.clear()
    eng.eval_acc.zero_()
    eng.eval_forward()
    assert XENT_CALLS == [512]                                # the logits GEMM's tile choice: the 2-CTA cluster
    after = (P.p32, P.m, P.v, P.g32, P.p16, eng.logits)
    assert all(torch.equal(x, y) for x, y in zip(before, after))
    import torch.nn.functional as TF

    ce = TF.cross_entropy
    monkeypatch.setattr(TF, "cross_entropy", lambda z, t: ce(z, t, reduction="none", ignore_index=-1))
    with torch.no_grad():
        want = ref(ins[0], ins[1], ins[2] if doc_mask else None)
    got = eng.losses
    valid = ins[1].reshape(-1) >= 0
    assert bool((got[~valid] == 0).all())
    err = float((got - want).abs().max())
    assert err < 5e-2, err                   # bf16 activations of the engine against the fp32 model
    assert float(eng.eval_acc[1]) == int(valid.sum())
    assert abs(float(eng.eval_acc[0]) - float(got.double().sum())) < 1e-6 * float(got.double().sum())
    # the training forward on the same batch: its loss differs only by the bf16 rounding of the logits
    eng.forward()
    assert float((eng.losses - got).abs().max()) < 5e-2


def test_eval_needs_the_wgmma_backend(monkeypatch):
    from trainingjob_operator_b200.models.gpt2 import GPT2Engine

    ke.install(monkeypatch)
    install_xent(monkeypatch)
    eng = GPT2Engine(_cfg(), 2, 128, "cpu", seed=3, gemm_backend="cublas")
    with pytest.raises(ValueError, match="wgmma"):
        eng.eval_forward()


def test_every_gemm_the_eval_forward_issues_has_a_kernel(monkeypatch, variants):  # noqa: F811
    """The eval forward's GEMMs -- the layers' and the cross-entropy logits GEMM -- all have compiled kernels, and all
    four tile configurations of the cross-entropy epilogue are compiled."""
    ke.install(monkeypatch)
    install_xent(monkeypatch)
    calls = set()
    gemm = F.gemm

    def rec_gemm(a, b, out, *, a_mn=False, b_mn=False, **kw):
        calls.add((bool(a_mn), bool(b_mn), F.gemm_epilogue(out, **{k: v for k, v in kw.items()
                                                                 if k not in ("split_k", "block_n", "max_ctas")})))
        return gemm(a, b, out, a_mn=a_mn, b_mn=b_mn, **kw)

    def rec_xent(x, w, *a, **kw):
        calls.add((False, False, F.EPI_XENT | F.EPI_OUT_F32))      # the library's key of the kernel it launches
        return gemm_xent(x, w, *a, **kw)

    monkeypatch.setattr(F, "gemm", rec_gemm)
    monkeypatch.setattr(F, "gemm_xent", rec_xent)
    from trainingjob_operator_b200.models.gpt2 import GPT2Engine

    eng = GPT2Engine(_cfg(), 2, 128, "cpu", seed=3)
    eng.eval_forward()
    assert (False, False, F.EPI_XENT | F.EPI_OUT_F32) in calls and (False, False, F.EPI_BIAS) in calls
    missing = {(a, b, F.epilogue_name(e)) for a, b, e in calls - _compiled_pairs(variants)}
    assert not missing, f"GEMMs without a compiled kernel: {missing}"


def test_the_cross_entropy_epilogue_keeps_the_logits_on_chip(variants):  # noqa: F811
    """All four tile configurations of EPI_XENT are compiled; each computes exponentials (MUFU.EX2), stores no tile by
    TMA (no UTMASTG) and uses no global reduction or atomic: the only global stores are plain stores of the partials
    and the target logits."""
    import re

    xent = {k: ops for k, ops in variants.items() if k[4] == F.EPI_XENT | F.EPI_OUT_F32}
    assert {(k[0], k[3]) for k in xent} == {(128, 1), (256, 1), (256, 2), (256, 4)}
    for k, ops in xent.items():
        assert "MUFU.EX2" in ops, k
        assert not [o for o in ops if o.startswith("UTMASTG")], k
        assert not [o for o in ops if re.match(r"(RED|ATOM)", o)], k


# ------------------------------------------------------------------------------------ 3. workers over gloo
WORKER = """
import os, sys, json, atexit
sys.path.insert(0, {root!r}); sys.path.insert(0, {tests!r})
import kernel_emulation as ke
ke.install()
import test_heldout_eval as th
th.install_xent()
from trainingjob_operator_b200.runtime import worker as W
RECORD = []
def build(args, device):
    ad = W.EngineAdapter(args.model, args.batch, args.seq, args, device="cpu")
    step = ad.train_step
    def recorded():
        loss = step()
        RECORD.append(loss)
        return loss
    ad.train_step = recorded
    return ad
W.build_adapter = build
atexit.register(lambda: json.dump(RECORD, open(os.path.join({out!r}, "steps%s.json" % os.environ["RANK"]), "w")))
sys.exit(W.main(sys.argv[1:]))
"""


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _run_workers(tmp_path, n, argv, tag):
    out = tmp_path / tag
    out.mkdir()
    script = out / "worker.py"
    script.write_text(textwrap.dedent(WORKER.format(root=ROOT, tests=TESTS, out=str(out))))
    port = _free_port()
    procs = []
    for r in range(n):
        env = dict(os.environ, RANK=str(r), WORLD_SIZE=str(n), LOCAL_RANK=str(r), MASTER_ADDR="127.0.0.1",
                   MASTER_PORT=str(port), OMP_NUM_THREADS="1", AITJ_WORKDIR=str(out), TRAININGJOB_NAME="ev")
        env.pop("AITJ_MASTER", None)
        procs.append(subprocess.Popen([sys.executable, str(script), "--cpu", "--result", str(out / "result.json"),
                                       "--dump-outputs", str(out / "dump")] + argv, env=env,
                                      stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True))
    logs = [p.communicate(timeout=900)[0] for p in procs]
    for p, log in zip(procs, logs):
        assert p.returncode == 0, log[-4000:]
    steps = [json.load(open(out / f"steps{r}.json")) for r in range(n)]
    return json.load(open(out / "result.json")), np.load(out / "dump" / "weights_sample.npy"), steps, logs[0]


@pytest.mark.slow
def test_evaluation_changes_no_training_step_and_is_the_same_at_any_world_size(tmp_path):
    """Two ranks, --global-batch 8 in micro-batches of 2, 4 steps, --eval-every 2 on 13 held-out windows: the same
    training losses and final weights, bit for bit, as without evaluation; the evaluations (before step 2 and after
    step 4) equal one rank's within 1e-6."""
    train = write_llmc(tmp_path / "train_000.bin", structured_corpus(60000, 1000, 999, 3))
    val = write_llmc(tmp_path / "val_000.bin", structured_corpus(20000, 1000, 999, 4))
    base = ["--model", "gpt2-tiny", "--batch", "2", "--seq", "128", "--steps", "3", "--warmup", "1", "--lr", "1e-4",
            "--data", train, "--global-batch", "8"]
    ev = ["--eval-data", val, "--eval-every", "2", "--eval-samples", "13"]
    r2, w2, s2, log = _run_workers(tmp_path, 2, base + ev, "w2eval")
    r2n, w2n, s2n, _ = _run_workers(tmp_path, 2, base, "w2")
    r1, _, _, _ = _run_workers(tmp_path, 1, base + ev, "w1eval")
    assert s2 == s2n and np.array_equal(w2, w2n)
    assert "evals" not in r2n
    assert [e["step"] for e in r2["evals"]] == [2, 4] and r2["eval_loss_last"] == r2["evals"][-1]["loss"]
    assert all(e["tokens"] == 13 * 128 and e["samples"] == 13 for e in r2["evals"])
    assert "eval loss" in log
    for a, b in zip(r2["evals"], r1["evals"]):
        assert abs(a["loss"] - b["loss"]) <= 1e-6 * abs(b["loss"]), (a, b)
    assert r2["evals"][0]["loss"] > r2["evals"][-1]["loss"] - 1.0 and np.isfinite(r2["eval_loss_last"])


RECOVERY_WORKER = """
import os, signal, sys
sys.path.insert(0, {root!r}); sys.path.insert(0, os.path.join({root!r}, "tests"))
import kernel_emulation as ke
ke.install()
import test_heldout_eval as th
th.install_xent()
from trainingjob_operator_b200.runtime import worker as W

def build(args, device):
    ad = W.EngineAdapter(args.model, args.batch, args.seq, args, device="cpu")
    evaluate, step = ad.evaluate, ad.train_step
    seen = []
    def evaluated(**kw):
        out = evaluate(**kw)
        seen.append(1)
        return out
    def train_step():
        # the first incarnation of rank 1 dies in the step right after its first evaluation
        if seen and os.environ.get("RANK") == "1" and os.environ.get("TRAININGJOB_REPLICA_RESTARTCOUNT", "0") == "0":
            os.kill(os.getpid(), signal.SIGKILL)
        return step()
    ad.evaluate, ad.train_step = evaluated, train_step
    return ad
W.build_adapter = build
sys.exit(W.main(sys.argv[1:]))
"""


@pytest.mark.slow
def test_a_peer_lost_right_after_an_evaluation_is_evaluated_again_by_every_rank(tmp_path):
    """A ``faultTolerant`` job of two engine workers (emulated kernels, gloo) submitted through ``LocalCluster``: rank 1
    dies in the training step right after the evaluation at step 2.  The survivor keeps its process and the replacement
    joins at step 2; both evaluate step 2 again -- the replacement has never evaluated it, so a survivor that went
    straight into the training step would meet the replacement's evaluation all-reduce with its gradient all-reduce --
    and the job runs to its end with the same evaluation loss at the repeated boundary."""
    import time

    from trainingjob_operator_b200.api import constants as C
    from trainingjob_operator_b200.cmd.local import LocalCluster
    from trainingjob_operator_b200.cmd.options import TrainingJobOperatorOption

    train = write_llmc(tmp_path / "train_000.bin", structured_corpus(60000, 1000, 999, 3))
    val = write_llmc(tmp_path / "val_000.bin", structured_corpus(20000, 1000, 999, 4))
    script = tmp_path / "worker_cpu.py"
    script.write_text(textwrap.dedent(RECOVERY_WORKER.format(root=ROOT)))
    # --steps 0: trains until the job is deleted, so only the --eval-every boundaries evaluate
    worker = [sys.executable, str(script), "--cpu", "--model", "gpt2-tiny", "--batch", "2", "--seq", "128", "--steps",
              "0", "--elastic", "--data", train, "--eval-data", val, "--eval-every", "2", "--eval-samples", "6",
              "--step-sleep", "0.05"]
    job = {"apiVersion": C.API_VERSION, "kind": C.KIND, "metadata": {"name": "ev"},
           "spec": {"frameworkType": "pytorch", "faultTolerant": True, "replicaSpecs": {"trainer": {
               "replicas": 2, "minReplicas": 1, "maxReplicas": 2, "edlPolicy": "Manual", "restartPolicy": "OnFailure",
               "restartLimit": 4,
               "template": {"spec": {"terminationGracePeriodSeconds": 1, "containers": [{
                   "name": "aitj-trainer", "command": worker, "workingDir": ROOT,
                   "env": [{"name": "PYTHONPATH", "value": ROOT}, {"name": "OMP_NUM_THREADS", "value": "2"}]}]}}}}}}
    pattern = re.compile(r"\[worker 0\] step (\d+): eval loss (\S+)")

    def log0():
        return open(os.path.join(lc.workdir, "logs", "default_ev-trainer-0_aitj-trainer.log")).read()

    with LocalCluster(num_gpus=0, workdir=str(tmp_path / "wd"), option=TrainingJobOperatorOption(thread_num=2)) as lc:
        try:
            lc.apply(job)
            t0 = time.time()
            evals = []
            while time.time() - t0 < 300:
                if os.path.exists(os.path.join(lc.workdir, "logs", "default_ev-trainer-0_aitj-trainer.log")):
                    evals = [(int(a), float(b)) for a, b in pattern.findall(log0())]
                    if [e[0] for e in evals][:4] == [2, 2, 4, 6]:
                        break
                time.sleep(0.2)
            log = log0()
            j = lc.jobs().get("ev")
        finally:
            lc.jobs().delete("ev")
            time.sleep(0.5)
    assert "lost a peer" in log and "keeping state" in log and "giving up" not in log, log[-3000:]
    assert j.status.restart_counts == {"trainer": 1}, j.status.restart_counts     # rank 0 was never restarted
    assert [e[0] for e in evals][:4] == [2, 2, 4, 6], (evals, log[-3000:])
    (_, first), (_, again) = evals[:2]
    assert abs(first - again) <= 1e-6 * abs(first), evals


# ------------------------------------------------------------------------------------ 4. refusals
def test_evaluation_is_refused_where_it_cannot_run(monkeypatch, tmp_path):
    from trainingjob_operator_b200.runtime.data import DataError
    from trainingjob_operator_b200.runtime.worker import EngineAdapter, parse_args

    for argv, what in ((["--model", "bert-tiny", "--eval-data", "x.bin"], "GPT-2 models only"),
                       (["--model", "gpt2-tiny", "--gemm", "cublas", "--eval-data", "x.bin"], "--gemm wgmma"),
                       (["--model", "gpt2-tiny", "--eval-every", "5"], "need --eval-data")):
        err = io.StringIO()
        monkeypatch.setattr(sys, "stderr", err)
        with pytest.raises(SystemExit):
            parse_args(argv)
        assert what in err.getvalue(), err.getvalue()
    monkeypatch.undo()
    ke.install(monkeypatch)
    install_xent(monkeypatch)
    val = write_llmc(tmp_path / "val_000.bin", structured_corpus(129 * 10 + 1, 1000, 999, 4))
    with pytest.raises(DataError, match="holds only 10 windows"):
        EngineAdapter("gpt2-tiny", 2, 128, _args(batch=2, eval_data=val, eval_samples=11), device="cpu")
    toks = structured_corpus(20000, 1000, 999, 4)
    toks[3000] = 1000                                           # outside gpt2-tiny's vocabulary
    bad = write_llmc(tmp_path / "val_bad.bin", toks)
    a = EngineAdapter("gpt2-tiny", 2, 128, _args(batch=2, eval_data=bad, eval_samples=40), device="cpu")
    a.trainer = types.SimpleNamespace(world=1, rank=0)
    with pytest.raises(DataError, match=r"val_bad\.bin: token id 1000 at token offset 3000"):
        list(a._eval_inputs())


# ------------------------------------------------------------------------------------ 5. reports
def _job(name, metrics):
    st = types.SimpleNamespace(phase="Running", rendezvous=None)
    return types.SimpleNamespace(name=name, status=st, annotations={"aitj.b200/metrics": json.dumps(metrics)})


def test_eval_loss_reaches_top_and_the_job_gauge():
    from trainingjob_operator_b200.cli.kubectl import CLI
    from trainingjob_operator_b200.controller.trainingjob import observe_worker_reports
    from trainingjob_operator_b200.utils import metrics

    jobs = [_job("with-eval", {"samples_per_sec": 100.0, "ms_per_step": 10.0, "steps_done": 8, "eval_loss": 3.25,
                               "eval_step": 8}),
            _job("no-eval", {"samples_per_sec": 50.0})]
    lister = types.SimpleNamespace(list=lambda: types.SimpleNamespace(items=jobs))
    cs = types.SimpleNamespace(elasticdeeplearning_v1=lambda: types.SimpleNamespace(aitrainingjobs=lambda ns: lister))
    out = io.StringIO()
    cli = CLI.__new__(CLI)
    cli.cs, cli.out = cs, out
    cli.p = lambda s="": out.write(s + "\n")
    assert cli.top("default", False) == 0
    lines = out.getvalue().splitlines()
    assert lines[0].split()[:4] == ["NAME", "PHASE", "WORLD", "SAMPLES/S"] and lines[0].rstrip().endswith("EVAL LOSS")
    assert lines[1].split()[0] == "with-eval" and lines[1].split()[-1] == "3.2500"
    assert lines[2].split()[0] == "no-eval" and lines[2].split()[-1] == "<none>"

    metrics.reset()
    base = {"metadata": {"namespace": "default", "name": "j", "annotations": {}}}
    cur = {"metadata": {"namespace": "default", "name": "j", "annotations": {
        "aitj.b200/metrics": json.dumps({"samples_per_sec": 10.0, "eval_loss": 2.5, "eval_step": 4})}}}
    observe_worker_reports(base, cur)
    assert 'aitj_job_eval_loss{job="j",namespace="default"} 2.5' in metrics.render()
    metrics.reset()


def test_the_final_report_carries_the_last_evaluation():
    from trainingjob_operator_b200.runtime.elastic import ElasticWatcher

    w = ElasticWatcher.__new__(ElasticWatcher)
    sent = {}
    w._annotate = lambda k, v: sent.update({k: v})
    w.report_result({"samples_per_sec": 1.0, "evals": [{"step": 2, "loss": 4.0}, {"step": 4, "loss": 3.5}]})
    m = sent["aitj.b200/metrics"]
    assert m["eval_loss"] == 3.5 and m["eval_step"] == 4
    w.report_result({"samples_per_sec": 1.0})
    assert "eval_loss" not in sent["aitj.b200/metrics"]


# ------------------------------------------------------------------------------------ GPU
def _run_case(name: str, timeout: int = 900):
    r = subprocess.run([sys.executable, "-m", "trainingjob_operator_b200.ops.selfcheck", "--case", name], cwd=ROOT,
                       capture_output=True, text=True, timeout=timeout)
    sys.stdout.write(r.stdout[-4000:])
    sys.stderr.write(r.stderr[-2000:])
    assert r.returncode == 0, f"selfcheck {name} failed:\n{r.stdout[-3000:]}\n{r.stderr[-1500:]}"


@pytest.mark.gpu
def test_gemm_xent_against_fp64_in_every_tile_configuration():
    _run_case("gemm_xent")


@pytest.mark.gpu
def test_gpt2_small_eval_forward_against_the_training_forward_and_the_fp32_model():
    _run_case("gpt2_eval")


def _worker(argv, timeout=900):
    env = dict(os.environ, WORLD_SIZE="1", RANK="0", PYTHONPATH=ROOT)
    env.pop("AITJ_MASTER", None)
    r = subprocess.run([sys.executable, "-m", "trainingjob_operator_b200.runtime.worker"] + argv, cwd=ROOT, env=env,
                       capture_output=True, text=True, timeout=timeout)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    return r.stdout


@pytest.mark.gpu
def test_one_gpu_worker_evaluates_a_held_out_shard(tmp_path):
    from trainingjob_operator_b200.runtime.elastic import ElasticWatcher

    train = write_llmc(tmp_path / "train_000.bin", structured_corpus(400000, 1000, 999, 0))
    val = write_llmc(tmp_path / "val_000.bin", structured_corpus(60000, 1000, 999, 7))
    res = str(tmp_path / "r.json")
    log = _worker(["--model", "gpt2-tiny", "--batch", "8", "--seq", "128", "--steps", "60", "--warmup", "3", "--lr",
                   "1e-3", "--data", train, "--eval-data", val, "--eval-every", "20", "--eval-samples", "100",
                   "--result", res])
    out = json.load(open(res))
    print(json.dumps({k: out[k] for k in ("loss_first", "loss_last", "ms_per_step", "evals")}))
    steps = [e["step"] for e in out["evals"]]
    assert steps == [20, 40, 60, 63], steps               # every 20 steps, and after the last of 3 + 60
    losses = [e["loss"] for e in out["evals"]]
    assert all(np.isfinite(losses)) and losses[-1] < losses[0], losses
    assert all(e["tokens"] == 100 * 128 for e in out["evals"]) and out["eval_loss_last"] == losses[-1]
    assert out["cuda_graph"] and not out["graph_error"]
    assert "eval loss" in log
    w = ElasticWatcher.__new__(ElasticWatcher)
    sent = {}
    w._annotate = lambda k, v: sent.update({k: v})
    w.report_result(out)
    assert sent["aitj.b200/metrics"]["eval_loss"] == losses[-1]


TWO_GPU_SCRIPT = """
import os, sys, json, torch, torch.distributed as dist
sys.path.insert(0, {root!r})
from trainingjob_operator_b200.runtime.worker import EngineAdapter, parse_args
rank = int(os.environ.get("RANK", "0"))
world = int(os.environ.get("WORLD_SIZE", "1"))
torch.cuda.set_device(rank)
if world > 1:
    dist.init_process_group("nccl", device_id=torch.device("cuda", rank))
args = parse_args(["--model", "gpt2-tiny", "--batch", "4", "--seq", "128", "--data", {train!r}, "--global-batch", "8",
                   "--lr", "1e-3", "--eval-data", {val!r}, "--eval-samples", "37"])
a = EngineAdapter("gpt2-tiny", 4, 128, args)
a.bind(None)
evals = [a.evaluate()]
for _ in range(4):
    a.train_step()
evals.append(a.evaluate())
json.dump(evals, open(os.path.join({out!r}, f"w{{world}}_{{rank}}.json"), "w"))
if world > 1:
    dist.destroy_process_group()
"""


@pytest.mark.gpu
@pytest.mark.gpu2
def test_two_gpus_evaluate_as_one(tmp_path):
    """37 held-out windows in micro-batches of 4 on 2 GPUs (5 + 5 micro-batches, the last one padded) and on one: the
    same evaluation losses before and after 4 training steps, within 1e-4 relative."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    train = write_llmc(tmp_path / "train_000.bin", structured_corpus(200000, 1000, 999, 2))
    val = write_llmc(tmp_path / "val_000.bin", structured_corpus(60000, 1000, 999, 3))
    script = tmp_path / "ev2.py"
    script.write_text(TWO_GPU_SCRIPT.format(root=ROOT, train=train, val=val, out=str(tmp_path)))
    port = _free_port()
    for world in (1, 2):
        procs = [subprocess.Popen([sys.executable, str(script)], cwd=ROOT, stdout=subprocess.PIPE,
                                  stderr=subprocess.STDOUT, text=True,
                                  env=dict(os.environ, RANK=str(r), WORLD_SIZE=str(world), MASTER_ADDR="127.0.0.1",
                                           MASTER_PORT=str(port + world)))
                 for r in range(world)]
        logs = [p.communicate(timeout=900)[0] for p in procs]
        assert all(p.returncode == 0 for p in procs), "\n".join(l[-3000:] for l in logs)
    one = json.load(open(tmp_path / "w1_0.json"))
    for r in range(2):
        two = json.load(open(tmp_path / f"w2_{r}.json"))
        for a, b in zip(two, one):
            assert a["tokens"] == b["tokens"] == 37 * 128
            assert abs(a["loss"] - b["loss"]) <= 1e-4 * abs(b["loss"]), (a, b)
    assert one[1]["loss"] < one[0]["loss"]
