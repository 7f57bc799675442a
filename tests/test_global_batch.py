"""A fixed global batch at any world size: the micro-batch plan (``runtime/accumulation.py``), gradient accumulation in
``EngineTrainer`` and ``TorchAdapter`` / ``FlatDDP``, the worker's ``--global-batch`` and its reports.

CPU tests run the engines with the kernel entry points emulated (``tests/kernel_emulation.py``) and gloo between
processes; the GPU tests run the hand-written kernels on an H100."""
import json
import os
import socket
import subprocess
import sys
import textwrap
import threading
import time
import types

import numpy as np
import pytest
import torch

import kernel_emulation as ke
from test_engine_launches import CONFIGS, ENTRY_POINTS, GOLDEN, _engine, _Recorder
from test_packed_documents import install_doc_attention, structured_corpus, write_llmc, write_raw
from trainingjob_operator_b200.runtime.accumulation import micro_batch_plan

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTS = os.path.dirname(os.path.abspath(__file__))


def rel(a, b):
    return float((a.float() - b.float()).norm() / (b.float().norm() + 1e-12))


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


# ------------------------------------------------------------------------------------ 1. the plan
@pytest.mark.parametrize("G,B,W", [(8, 2, 1), (8, 2, 2), (8, 2, 3), (8, 2, 4), (8, 2, 5), (8, 2, 7), (12, 3, 2),
                                   (12, 3, 3), (6, 2, 4), (30, 5, 4), (64, 16, 8), (16, 16, 3), (48, 4, 5)])
def test_plan_covers_the_global_batch_once_and_balances_the_ranks(G, B, W):
    plans = [micro_batch_plan(G, B, W, r) for r in range(W)]
    k = G // B
    assert all(p.k == k and p.global_batch == G for p in plans)
    assert max(p.n for p in plans) - min(p.n for p in plans) <= 1
    assert all(p.n == (k + W - 1 - r) // W for r, p in enumerate(plans))     # ceil or floor of k / W; 0 when r >= k
    for pos in (0, 17, 1000):
        samples = sorted(s for p in plans for first, n in p.windows(pos) for s in range(first, first + n))
        assert samples == list(range(pos, pos + G))
    assert plans[0].accumulates == (k != W)


def test_plan_default_is_one_micro_batch_per_rank_and_bad_sizes_are_refused():
    for W in (1, 2, 5):
        for r in range(W):
            p = micro_batch_plan(0, 4, W, r)
            assert p.global_batch == 4 * W and p.n == 1 and not p.accumulates
            assert p.windows(100) == [(100 + 4 * r, 4)] and not p.fixed
            given = micro_batch_plan(4 * W, 4, W, r)
            assert (given.micro, given.k, given.accumulates, given.fixed) == (p.micro, p.k, False, True)
    with pytest.raises(ValueError):
        micro_batch_plan(10, 4, 1, 0)


class _StubTrainer:
    """The trainer as the adapter's data path sees it: the plan, and one loss per step."""

    def __init__(self, G, B, world, rank):
        self.world, self.rank, self.step_count = world, rank, 0
        self.plan = micro_batch_plan(G, B, world, rank)

    def step(self, *host):
        self.step_count += 1
        return 0.0

    def accumulate(self, micro_inputs):
        n = sum(1 for _ in micro_inputs)
        assert n == self.plan.n
        self.step_count += 1
        return 0.0


def _adapter_on(data, G, B, world, rank, position):
    from trainingjob_operator_b200.runtime.worker import EngineAdapter

    a = EngineAdapter.__new__(EngineAdapter)
    a.data, a.batch, a.data_position = data, B, position
    a.trainer = _StubTrainer(G, B, world, rank)
    return a


def _read(a):
    a.train_step()
    return getattr(a, "samples_read", None) or a.data.samples_read


def test_default_global_batch_reads_what_each_rank_read_before(tmp_path):
    """G = W*B: rank r reads [pos + r*B, pos + (r+1)*B) through the single-micro-batch path, as without the flag."""
    from trainingjob_operator_b200.runtime.data import TokenFileData

    write_raw(tmp_path / "c.bin", np.arange(20000) % 1000)
    B = 3
    for world in (1, 2, 3):
        for r in range(world):
            d = TokenFileData(str(tmp_path / "c.bin"), 32, 1000, pin=False)
            a = _adapter_on(d, world * B, B, world, r, 30)
            assert _read(a) == list(range(30 + r * B, 30 + (r + 1) * B))
            assert a.data_position == 30 + world * B


def test_a_fixed_global_batch_reads_every_sample_once_across_rescales(tmp_path):
    """G = 4B through world sizes 2, 3 (uneven), 1 and 5 (an idle rank): every step covers [pos, pos + G) exactly once,
    the position advances by G, and the rescales leave no gap and no repeat."""
    from trainingjob_operator_b200.runtime.data import TokenFileData

    write_raw(tmp_path / "c.bin", np.arange(40000) % 1000)
    B, G = 3, 12
    pos, seen = 0, []
    for world, steps in ((2, 2), (3, 2), (1, 1), (5, 2)):
        for _ in range(steps):
            step = []
            for r in range(world):
                d = TokenFileData(str(tmp_path / "c.bin"), 32, 1000, pin=False)
                a = _adapter_on(d, G, B, world, r, pos)
                got = _read(a) if a.trainer.plan.n else (a.train_step(), [])[1]
                assert got == [s for first, n in a.trainer.plan.windows(pos) for s in range(first, first + n)]
                step += got
                assert a.data_position == pos + G
            assert sorted(step) == list(range(pos, pos + G))
            seen += step
            pos += G
    assert sorted(seen) == list(range(len(seen))) and len(seen) == G * 7


# ------------------------------------------------------------------------------------ 2. engine equivalence
GPT2_NAMES = ("wte", "wpe", "h0.qkv_w", "h0.qkv_b", "h0.proj_w", "h0.fc_w", "h0.fc_b", "h0.fc2_w", "h1.ln1_w", "h1.ln2_b",
              "h1.fc2_w", "lnf_w", "lnf_b")
BERT_NAMES = ("wte", "wpe", "wtt", "emb_ln_w", "h0.qkv_w", "h0.qkv_b", "h0.proj_w", "h0.fc_w", "h0.fc2_b", "h1.ln2_b",
              "mlm_w", "mlm_b", "mlm_ln_w")


def _perturb(eng, seed=9):
    g = torch.Generator().manual_seed(seed)
    for s_ in eng.params.specs:
        if len(s_.shape) == 1:
            eng.params.w32(s_.name).add_(torch.randn(s_.shape, generator=g) * 0.05)
    if "dec_b" in eng.params.by_name:
        eng.params.w32("dec_b")[eng.cfg.vocab_size:].zero_()
    eng.params.refresh_compute_copy()


def _model(model, B):
    """(engine of micro-batch B, micro-batch inputs of 4 micro-batches, joint inputs, reference-model loss fn)."""
    if model == "gpt2":
        from trainingjob_operator_b200.models.gpt2 import GPT2Config, GPT2Engine, GPT2Reference

        cfg = GPT2Config(vocab_size=1000, n_layer=2, n_head=4, n_embd=256, block_size=128, name="t")
        mk = lambda b: GPT2Engine(cfg, b, 128, "cpu", seed=3, gemm_backend="wgmma")      # noqa: E731
        tok = torch.randint(0, cfg.vocab_size, (4 * B, 128), generator=torch.Generator().manual_seed(5))
        tgt = torch.roll(tok, -1, dims=1)
        micro = [(tok[j * B:(j + 1) * B].reshape(-1), tgt[j * B:(j + 1) * B].reshape(-1)) for j in range(4)]
        joint = (tok.reshape(-1), tgt.reshape(-1))
        return cfg, mk, micro, joint, (lambda ref: ref(tok, tgt)), GPT2Reference, GPT2_NAMES
    from trainingjob_operator_b200.models.bert import BertConfig, BertEngine, BertReference, SyntheticMLM

    cfg = BertConfig.tiny()
    mk = lambda b: BertEngine(cfg, b, 128, "cpu", seed=3)       # noqa: E731
    data = SyntheticMLM(cfg.vocab_size, B, 128, n_batches=4, seed=5, pin=False)
    micro = [data.next() for _ in range(4)]
    joint = tuple(torch.cat([m[i] for m in micro]) for i in range(3))
    return cfg, mk, micro, joint, (lambda ref: ref(*(t.view(4 * B, 128) for t in joint))), BertReference, BERT_NAMES


@pytest.mark.parametrize("model", ["gpt2", "bert"])
def test_four_accumulated_micro_batches_equal_one_engine_on_the_joint_batch(monkeypatch, model):
    """k = 4 micro-batches of B through ``EngineTrainer.accumulate``: before the optimizer the gradient buffer divided by
    k equals (a) the gradient of one engine of batch 4B on the same samples, to reordered-sum rounding, and (b) the fp32
    reference model's on the joint batch, to bf16 rounding.  After the step the master weights equal the joint engine's.
    (BERT normalises each micro-batch by its own masked count: the step's gradient is a mean of per-micro-batch means.)"""
    from trainingjob_operator_b200.runtime.trainer import EngineTrainer

    ke.install(monkeypatch)
    B = 2
    cfg, mk, micro, joint, ref_loss, Ref, names = _model(model, B)
    acc, one = mk(B), mk(4 * B)
    _perturb(acc)
    _perturb(one)
    if model == "bert":
        # every synthetic micro-batch masks the same number of positions: a joint engine normalised by 4 times that
        # number computes the mean of the per-micro-batch means (with its own count it would divide by round(0.15 * 4BT))
        one.n_masked = 4 * acc.n_masked
    tr = EngineTrainer(acc, lr=1e-3, use_graph=False, global_batch=4 * B)
    tr1 = EngineTrainer(one, lr=1e-3, use_graph=False)
    assert tr.plan.k == 4 and tr.plan.n == 4 and tr.plan.accumulates and not tr1.plan.accumulates
    grads = {}
    for t, key in ((tr, "acc"), (tr1, "one")):
        real = t._optimizer

        def snap(real=real, t=t, key=key):
            grads[key] = t.engine.params.g32.clone() / t.plan.k
            real()

        t._optimizer = snap
    forwards = []
    real_fwd = acc.forward
    acc.forward = lambda: (forwards.append(1), real_fwd())[1]
    loss_acc = tr.accumulate(iter(micro))
    loss_one = tr1.step(*joint)
    assert len(forwards) == 4
    assert rel(grads["acc"], grads["one"]) < 1e-4, rel(grads["acc"], grads["one"])
    assert abs(loss_acc - loss_one) < 1e-4 * abs(loss_acc)
    assert rel(acc.params.p32, one.params.p32) < 1e-5          # after the step: the same master weights
    assert float(acc.params.g32.abs().max()) == 0.0 and float(tr.loss_sum.abs().max()) == 0.0
    # (b) against the fp32 reference, on fresh weights
    fresh = mk(4 * B)
    _perturb(fresh)
    ref = Ref(cfg, fresh.params)
    loss = ref_loss(ref)
    loss.backward()
    by = {s.name: s for s in acc.params.specs}
    for name in names:
        s = by[name]
        got = grads["acc"][s.offset:s.offset + s.numel].view(s.shape)
        assert rel(got, ref.p(name).grad) < 6e-2, name


# (k a power of two: the joint engine's loss scale 1 / (k B T) then rounds dlogits to bf16 exactly as 1 / (B T) does)
@pytest.mark.parametrize("world,k", [(3, 4), (3, 2)], ids=["uneven", "idle-rank"])
def test_owner_sharded_accumulation_equals_one_replica_on_the_joint_batch(monkeypatch, world, k):
    """The owner-sharded mode (``rs``) with its peer-memory kernels emulated, ranks as threads: every micro-batch's
    gradients are added into their owner's copy, and a rank with fewer (or no) micro-batches meets the others at the same
    device barriers.  After two steps each rank's shard of the master weights equals that of ONE engine that trained the
    joint batch of k micro-batches, and nothing is left in any gradient buffer."""
    from trainingjob_operator_b200.models.gpt2 import GPT2Config, GPT2Engine
    from trainingjob_operator_b200.runtime.trainer import EngineTrainer

    ke.install(monkeypatch)
    cfg = GPT2Config(vocab_size=1000, n_layer=2, n_head=4, n_embd=256, block_size=128, name="t")
    B, T, STEPS = 2, 128, 2
    g = torch.Generator().manual_seed(11)
    toks = [torch.randint(0, cfg.vocab_size, (k * B, T), generator=g) for _ in range(STEPS)]

    def inputs(step, j):
        t = toks[step][j * B:(j + 1) * B]
        return t.reshape(-1), torch.roll(t, -1, dims=1).reshape(-1)

    ref = GPT2Engine(cfg, k * B, T, "cpu", seed=3, gemm_backend="wgmma")
    _perturb(ref)
    tref = EngineTrainer(ref, lr=1e-3, use_graph=False)
    tref.max_norm = 0.5
    for step in range(STEPS):
        tref.step(toks[step].reshape(-1), torch.roll(toks[step], -1, dims=1).reshape(-1))

    fw = ke.FakeWorld(world)
    monkeypatch.setitem(ke._CURRENT, "world", fw)
    trainers = []
    for r in range(world):
        e = GPT2Engine(cfg, B, T, "cpu", seed=3, gemm_backend="wgmma")
        _perturb(e)
        tr = EngineTrainer(e, lr=1e-3, use_graph=False)
        tr.max_norm = 0.5
        # what the constructor sets up for the owner-sharded arm on a device with peer memory
        tr.world, tr.rank, tr.shard = world, r, fw.attach(e.params)
        tr.plan = micro_batch_plan(k * B, B, world, r)
        trainers.append(tr)
    assert [t.plan.n for t in trainers] == [len(range(r, k, world)) for r in range(world)]
    errors = []

    def rank_main(r):
        try:
            tr = trainers[r]
            for step in range(STEPS):
                tr.accumulate(inputs(step, j) for j in tr.plan.micro)
        except Exception as ex:  # noqa: BLE001
            errors.append((r, repr(ex)))
            fw.sync.abort()

    threads = [threading.Thread(target=rank_main, args=(r,)) for r in range(world)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(600)
    assert not errors, errors
    total = ref.params.total
    for r, tr in enumerate(trainers):
        sh = fw.shards[r]
        assert sh.barriers == 3 * STEPS                                   # the same barriers on every rank
        assert float(sh.g[:total].abs().max()) == 0.0 and float(tr.engine.params.g_small.abs().max()) == 0.0
        own = slice(sh.lo, sh.hi)
        assert rel(tr.engine.params.p32[own], ref.params.p32[own]) < 1e-4, r      # reordered sums, 2 AdamW steps
        assert torch.equal(tr.engine.params.p16, trainers[0].engine.params.p16)


# ------------------------------------------------------------------------------------ 3. the default path
def _normalise(calls):
    """The optimizer scalars the trainer passes differently from a bare ``optimizer_step`` (schedule on the device,
    step counter, world-size divisor)."""
    out = []
    for name, args in calls:
        if name == "adamw":
            args = dict(args, dyn=None, step=1, grad_div=1.0)
        out.append([name, args])
    return out


def _trainer_trace(name, mp, global_batch):
    from trainingjob_operator_b200.runtime.trainer import EngineTrainer
    from trainingjob_operator_b200.ops import functional as F

    model, kw, env, sharded = CONFIGS[name]
    install_doc_attention(mp)
    for key in ("AITJ_ATTN", "AITJ_ATTN_BWD", "AITJ_GEMM_PAIR", "AITJ_GEMM_CFG", "AITJ_WGRAD_STREAM"):
        mp.delenv(key, raising=False)
    for key, v in env.items():
        mp.setenv(key, v)
    world = 2 if sharded else 1
    engs = [_engine(model, kw) for _ in range(world)]
    trainers = []
    if sharded:
        fw = ke.FakeWorld(2)
        mp.setitem(ke._CURRENT, "world", fw)
    for r, e in enumerate(engs):
        tr = EngineTrainer(e, lr=1e-3, use_graph=False)
        if sharded:
            tr.world, tr.rank, tr.shard = world, r, fw.attach(e.params)
        tr.plan = micro_batch_plan(global_batch(e.B, world), e.B, world, r)
        trainers.append(tr)
    errors, rec = [], []

    def run(tr, record):
        try:
            host = [t.clone() for t in tr.engine.input_tensors()]
            step = (lambda: tr.accumulate(iter([host]))) if tr.plan.accumulates else (lambda: tr.step(*host))
            step()
            if record:
                rec.append(_Recorder(tr.engine))
                for n in ENTRY_POINTS:
                    mp.setattr(F, n, rec[0].wrap(n, getattr(F, n)))
            step()
        except Exception as ex:  # noqa: BLE001
            errors.append(repr(ex))
            if sharded:
                fw.sync.abort()

    threads = [threading.Thread(target=run, args=(tr, r == 0)) for r, tr in enumerate(trainers)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(600)
    assert not errors, errors
    return rec[0].calls


@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_global_batch_of_world_times_batch_issues_the_recorded_launches(monkeypatch, name):
    """G = W*B is today's step: the trainer launches exactly the recorded forward, backward and optimizer."""
    with open(GOLDEN) as f:
        want = json.load(f)[name]
    got = _normalise(_trainer_trace(name, monkeypatch, lambda B, W: W * B))
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, f"launch {i} of {len(want)} differs:\n got  {g}\n want {w}"
    assert len(got) == len(want)


# ------------------------------------------------------------------------------------ 4. hooks and collectives
class _LogReducer:
    def __init__(self, log):
        self.log = log

    def hook(self, name):
        self.log.append(("hook", name))

    def wait(self):
        self.log.append(("wait",))


class _ReplayGraph:
    """A captured graph segment as the trainer replays it, run eagerly."""

    def __init__(self, fn):
        self.fn = fn

    def replay(self):
        self.fn()


@pytest.mark.parametrize("mode", ["eager", "segments"])
def test_bucket_hooks_fire_only_on_the_last_micro_batch_and_an_idle_rank_issues_the_same(monkeypatch, mode):
    """NCCL bucketed mode at world 3, eagerly and as replayed graph segments.  Rank 0 with k = 5 runs two micro-batches:
    its bucket hooks (= all-reduces) fire only during the last one.  Rank 2 with k = 2 has no micro-batch: it issues the
    same hooks in the same order, the join, then the optimizer."""
    from trainingjob_operator_b200.runtime.trainer import EngineTrainer

    ke.install(monkeypatch)
    from trainingjob_operator_b200.models.gpt2 import GPT2Config, GPT2Engine

    cfg = GPT2Config(vocab_size=1000, n_layer=2, n_head=4, n_embd=256, block_size=128, name="t")
    seqs = {}
    for rank, k in ((0, 5), (2, 2)):
        e = GPT2Engine(cfg, 2, 128, "cpu", seed=3, gemm_backend="wgmma")
        tr = EngineTrainer(e, lr=1e-3, use_graph=False)
        log = []
        tr.world, tr.rank, tr.segmented = 3, rank, True
        tr.reducer = _LogReducer(log)
        e.grad_hook = tr.reducer.hook
        e.segment_join = True
        tr.plan = micro_batch_plan(k * 2, 2, 3, rank)
        real_fwd, real_opt = e.forward, tr._optimizer
        e.forward = lambda real_fwd=real_fwd, log=log: (log.append(("fwd",)), real_fwd())[1]
        tr._optimizer = lambda real_opt=real_opt, log=log: (log.append(("opt",)), real_opt())[1]
        if mode == "segments":
            parts = [((), e.forward)] + list(e.backward_segments()) + [(None, tr._optimizer)]
            tr.seg_graphs = [(b, _ReplayGraph(fn)) for b, fn in parts]
        host = [t.clone() for t in e.input_tensors()]
        tr.accumulate(iter([host] * tr.plan.n))
        seqs[rank] = log
    r0, idle = seqs[0], seqs[2]
    assert [x for x in r0 if x[0] == "fwd"] == [("fwd",)] * 2
    last_fwd = max(i for i, x in enumerate(r0) if x[0] == "fwd")
    assert all(x[0] != "hook" for x in r0[:last_fwd])                     # nothing reduced before the last micro-batch
    coll = [x for x in r0 if x[0] != "fwd"]
    assert [x for x in idle if x[0] != "fwd"] == coll and ("fwd",) not in idle
    assert coll[-2:] == [("wait",), ("opt",)] and len([x for x in coll if x[0] == "hook"]) >= 3


def test_eager_overlap_hooks_hold_back_until_the_last_micro_batch_and_an_idle_rank_reduces_every_bucket(monkeypatch):
    """``TorchAdapter`` with per-parameter post-accumulate hooks (the CPU / eager overlap mode): with k = 3 at world 2, rank
    0's two micro-batches start bucket reductions only during the second backward; rank 1 at world 4 (k = 1, idle)
    reduces every bucket, in bucket order, like a rank that had nothing to add."""
    from trainingjob_operator_b200.runtime.worker import TorchAdapter

    args = types.SimpleNamespace(seed=0, lr=1e-2, no_graph=True, global_batch=0)
    logs = {}
    for rank, world, k in ((0, 2, 3), (1, 4, 1)):
        a = TorchAdapter("mlp", 8, args, torch.device("cpu"))
        a.bind(None)
        log = []
        ddp = a.ddp
        ddp.world, ddp.reducer = world, _LogReducer(log)
        ddp.buckets = ddp.buckets or [("b0", 0, ddp.total)]
        for idx, p in enumerate(ddp.params):
            p.register_post_accumulate_grad_hook(ddp._make_hook(idx))
        a.plan = micro_batch_plan(k * 8, 8, world, rank)
        ddp.k = a.plan.k
        real = a._fwd_bwd
        a._fwd_bwd = lambda real=real, log=log: (log.append(("fwd",)), real())[1]
        a.train_step()
        logs[rank] = log
    r0, idle = logs[0], logs[1]
    fwds = [i for i, x in enumerate(r0) if x == ("fwd",)]
    assert len(fwds) == 2 and all(x[0] != "hook" for x in r0[:fwds[1]])
    assert [x[1] for x in r0 if x[0] == "hook"] and ("fwd",) not in idle
    nb = len(a.ddp.buckets)
    assert idle == [("hook", f"b{b}") for b in range(nb)] + [("wait",)]
    assert sorted(x[1] for x in r0 if x[0] == "hook") == sorted(f"b{b}" for b in range(nb))


# ------------------------------------------------------------------------------------ 5. workers over gloo
RECORDING_WORKER = """
import os, sys, json, atexit
sys.path.insert(0, {root!r}); sys.path.insert(0, {tests!r})
import kernel_emulation as ke
ke.install()
from trainingjob_operator_b200.runtime import worker as W
RECORD = []
_build = W.build_adapter
def build(args, device):
    import torch
    torch.manual_seed(args.seed)          # nn.Module initialisation from the global generator: the same at every W
    if args.model in ("gpt2-tiny", "bert-tiny"):
        ad = W.EngineAdapter(args.model, args.batch, args.seq, args, device="cpu")
    else:
        ad = _build(args, device)
    step = ad.train_step
    def recorded():
        loss = step()
        RECORD.append([loss, ad.plan.n, ad.plan.k])
        return loss
    ad.train_step = recorded
    return ad
W.build_adapter = build
atexit.register(lambda: json.dump(RECORD, open(os.path.join({out!r}, "steps%s.json" % os.environ["RANK"]), "w")))
sys.exit(W.main(sys.argv[1:]))
"""


def _run_recording_workers(tmp_path, n, argv, tag):
    out = tmp_path / tag
    out.mkdir()
    script = out / "worker.py"
    script.write_text(textwrap.dedent(RECORDING_WORKER.format(root=ROOT, tests=TESTS, out=str(out))))
    port = _free_port()
    procs = []
    for r in range(n):
        env = dict(os.environ, RANK=str(r), WORLD_SIZE=str(n), LOCAL_RANK=str(r), MASTER_ADDR="127.0.0.1",
                   MASTER_PORT=str(port), OMP_NUM_THREADS="1", AITJ_WORKDIR=str(out), TRAININGJOB_NAME="gb")
        env.pop("AITJ_MASTER", None)
        procs.append(subprocess.Popen([sys.executable, str(script), "--cpu", "--result", str(out / "result.json"),
                                       "--dump-outputs", str(out / "dump")] + argv, env=env,
                                      stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True))
    logs = [p.communicate(timeout=900)[0] for p in procs]
    for p, log in zip(procs, logs):
        assert p.returncode == 0, log[-4000:]
    steps = [json.load(open(out / f"steps{r}.json")) for r in range(n)]
    # the job's loss of a step: the mean over its k micro-batches, from each rank's mean over its own
    job_losses = [sum(s[i][0] * s[i][1] for s in steps if s[i][1]) / steps[0][i][2] for i in range(len(steps[0]))]
    return (json.load(open(out / "result.json")), np.load(out / "dump" / "weights_sample.npy"), np.asarray(job_losses),
            steps)


# The runs differ only in the order in which the k micro-batch gradients are summed (one buffer, or per rank and then
# all-reduced), ~1e-7 relative in fp32 per element.  AdamW normalises each element by its own gradient history, so an
# element whose summed gradient nearly cancels moves by a fraction of lr in a direction set by that rounding: the worst
# element is no measure, the norm of the difference of all master weights is.  Measured in the emulation: ~1e-4 of the
# weights' norm after 3 steps at lr 1e-3 (within 1e-5 for the single step of the engine test above); the bound is 10x.
WEIGHT_TOL, LOSS_TOL = 1e-3, 1e-4


@pytest.mark.slow
@pytest.mark.parametrize("model", ["gpt2-tiny", "mlp"])
def test_workers_at_world_sizes_1_2_3_and_5_follow_the_same_trajectory(tmp_path, model):
    """``--global-batch 4B`` at W = 1, 2, 3 (uneven: 2/1/1), 4 (k = W: one micro-batch per rank) and 5 (rank 4 idle):
    the same master weights and per-step job losses; ``data_position = steps * G`` on a token shard."""
    B = 2 if model == "gpt2-tiny" else 8
    argv = ["--model", model, "--batch", str(B), "--steps", "2", "--warmup", "1", "--global-batch", str(4 * B)]
    if model == "gpt2-tiny":
        shard = write_llmc(tmp_path / "train_000.bin", structured_corpus(60000, 1000, 999, 3))
        argv += ["--seq", "128", "--data", shard, "--lr", "1e-3"]
    else:
        argv += ["--lr", "1e-2"]
    runs = {W: _run_recording_workers(tmp_path, W, argv, f"w{W}") for W in (1, 2, 3, 4, 5)}
    r1, w1, l1, _ = runs[1]
    for W, (r, w, losses, steps) in runs.items():
        assert r["global_batch"] == 4 * B and r["micro_batches"] == 4 and r["world"] == W, r
        assert r["micro_batches_this_rank"] == len(range(0, 4, W))
        assert [s[0][1] for s in steps] == [len(range(rk, 4, W)) for rk in range(W)]
        if model == "gpt2-tiny":
            assert r["data_position"] == 3 * 4 * B
        dw, dl = float(np.linalg.norm(w - w1) / np.linalg.norm(w1)), float(np.abs(losses - l1).max() / np.abs(l1).max())
        print(f"{model} W={W}: weights {dw:.2e}, losses {dl:.2e} (relative to W=1)")
        assert dw < WEIGHT_TOL and dl < LOSS_TOL, (W, dw, dl, losses, l1)
    if W == 5:
        assert all(np.isnan(s[0]) for s in runs[5][3][4])             # rank 4 trained nothing and says so


# ------------------------------------------------------------------------------------ 7. refusals and the stall breaker
def test_worker_refuses_a_global_batch_it_cannot_serve(monkeypatch):
    from trainingjob_operator_b200.runtime.worker import parse_args

    assert parse_args(["--batch", "4", "--global-batch", "12"]).global_batch == 12
    assert parse_args([]).global_batch == 0
    with pytest.raises(SystemExit):
        parse_args(["--batch", "4", "--global-batch", "10"])
    monkeypatch.setenv("AITJ_ALLREDUCE", "mc")
    with pytest.raises(SystemExit):
        parse_args(["--batch", "4", "--global-batch", "8"])
    assert parse_args(["--batch", "4"]).global_batch == 0            # mc without the flag is today's path


def test_stall_breaker_patience_follows_the_steps_of_the_generation():
    """The bookkeeping the worker loop does around every step (``begin_step`` at the step boundary, ``step_done`` after a
    completed step): the first step of a generation gets the first-step patience; the second twice the first step (which
    also captured graphs, so it bounds a steady step); from then on twice the slowest steady step; ``after_s`` at least.
    A new generation starts over.  ResNet-50 at B = 128 accumulating 32 micro-batches: a 40 s first step and 10 s steady
    steps give the second step 80 s and the later ones 20 s, not the bare 3 s."""
    from trainingjob_operator_b200.runtime import rendezvous as R

    br = R.StallBreaker(types.SimpleNamespace(fetch_now=lambda: None), 3.0)
    try:
        seen = []
        for gen, secs in ((1, 40.0), (1, 10.0), (1, 9.0), (1, 12.0), (2, 5.0), (2, 0.1), (2, 0.2)):
            br.begin_step(gen)
            seen.append(br.patience)
            br.step_done(gen, secs)
        br.begin_step(2)
        seen.append(br.patience)
        br.begin_step(3)
        seen.append(br.patience)
        assert seen == [30.0, 80.0, 20.0, 20.0, 30.0, 10.0, 3.0, 3.0, 30.0], seen
    finally:
        br.stop()


def test_stall_breaker_waits_for_a_slow_healthy_step_and_still_trips_on_a_stuck_one(monkeypatch):
    """A newer generation is pending throughout.  After a capture step and one steady step of 1.5 s (the threshold is
    0.5 s) the patience is 3 s: another 1.6 s step is not aborted; a step that does not end is."""
    from trainingjob_operator_b200.runtime import rendezvous as R

    aborted = []
    monkeypatch.setattr(R.dist, "is_initialized", lambda: True)
    monkeypatch.setattr(R, "teardown_group", lambda broken=False: aborted.append(time.time()))
    watcher = types.SimpleNamespace(fetch_now=lambda: {"generation": 2})
    br = R.StallBreaker(watcher, 0.5)
    try:
        br.step_done(1, 0.2)
        br.step_done(1, 1.5)
        br.begin_step(1)
        assert br.patience == 3.0
        br.progress(1)
        br.in_step = True
        time.sleep(1.6)                                   # a healthy accumulated step, longer than after_s
        br.in_step = False
        assert not br.tripped and not aborted
        br.progress(1)
        br.in_step = True
        t0 = time.time()
        while not br.tripped and time.time() - t0 < 10:
            time.sleep(0.05)
        assert br.tripped and aborted and aborted[0] - t0 >= 2.9
    finally:
        br.in_step = False
        br.stop()


class _NoCuda:
    """Just enough of ``torch.cuda`` for ``EngineTrainer._warm_up`` on the CPU: streams that run in line."""

    class Stream:
        def wait_stream(self, other):
            pass

    @staticmethod
    def stream(s):
        import contextlib

        return contextlib.nullcontext()

    @staticmethod
    def current_stream():
        return _NoCuda.Stream()

    @staticmethod
    def synchronize():
        pass


@pytest.mark.parametrize("k", [1, 2], ids=["k-equals-world", "accumulating"])
def test_graph_warm_up_leaves_no_mark_with_a_fixed_global_batch(monkeypatch, k):
    """Before capturing its graphs a trainer runs two complete steps (optimizer included).  With ``--global-batch`` it
    puts the state back afterwards -- also at a world size where the step is one micro-batch (k = W), the trainer's
    single-micro-batch path -- so a trainer that warmed up follows the trajectory of one that did not.  Without the flag
    the warm-up keeps its updates, as it always did."""
    from trainingjob_operator_b200.runtime import trainer as TR

    ke.install(monkeypatch)
    cfg, mk, micro, _, _, _, _ = _model("gpt2", 2)
    monkeypatch.setattr(TR.torch, "cuda", _NoCuda)
    runs = {}
    for name, G, warm in (("fixed+warm-up", 2 * k, True), ("fixed", 2 * k, False), ("default+warm-up", 0, True)):
        if G == 0 and k != 1:
            continue
        e = mk(2)
        _perturb(e)
        tr = TR.EngineTrainer(e, lr=1e-3, use_graph=False, global_batch=G)
        assert tr.plan.accumulates == (k != 1) and tr.plan.fixed == bool(G)
        for step in range(2):
            inputs = micro[step * k:(step + 1) * k]
            for dst, src in zip(e.input_tensors(), inputs[0]):
                dst.copy_(src)
            if warm and step == 0:
                e.set_step_scalars(TR.cosine_lr(1, tr.lr), 1)     # as step() does before it captures
                tr._warm_up()
                assert float(e.params.g32.abs().max()) == 0.0 and float(tr.loss_sum.abs().max()) == 0.0
            if tr.plan.accumulates:
                tr.accumulate(iter(inputs))
            else:
                tr.step(*inputs[0])
        runs[name] = e.params.p32.clone()
    assert torch.equal(runs["fixed+warm-up"], runs["fixed"])
    if k == 1:
        assert rel(runs["default+warm-up"], runs["fixed"]) > 1e-3          # the default path's warm-up is unchanged


# ------------------------------------------------------------------------------------ GPU
def _run_case(name: str, timeout: int = 600):
    r = subprocess.run([sys.executable, "-m", "trainingjob_operator_b200.ops.selfcheck", "--case", name], cwd=ROOT,
                       capture_output=True, text=True, timeout=timeout)
    sys.stdout.write(r.stdout[-4000:])
    sys.stderr.write(r.stderr[-2000:])
    assert r.returncode == 0, f"selfcheck {name} failed:\n{r.stdout[-3000:]}\n{r.stderr[-1500:]}"


@pytest.mark.gpu
def test_engines_accumulate_on_the_wgmma_path_in_one_graph():
    _run_case("accumulation")


def _worker(argv, timeout=900):
    env = dict(os.environ, WORLD_SIZE="1", RANK="0", PYTHONPATH=ROOT)
    env.pop("AITJ_MASTER", None)
    r = subprocess.run([sys.executable, "-m", "trainingjob_operator_b200.runtime.worker"] + argv, cwd=ROOT, env=env,
                       capture_output=True, text=True, timeout=timeout)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]


@pytest.mark.gpu
def test_one_gpu_worker_accumulates_in_cuda_graphs(tmp_path):
    shard = write_llmc(tmp_path / "train_000.bin", structured_corpus(400000, 1000, 999, 0))
    res = str(tmp_path / "r.json")
    _worker(["--model", "gpt2-tiny", "--batch", "8", "--seq", "128", "--steps", "60", "--warmup", "3", "--lr", "1e-3",
             "--data", shard, "--global-batch", "32", "--result", res])
    out = json.load(open(res))
    print(json.dumps({k: out[k] for k in ("loss_first", "loss_last", "ms_per_step", "samples_per_sec", "data_position")}))
    assert out["cuda_graph"] and not out["graph_error"]
    assert out["global_batch"] == 32 and out["micro_batches"] == 4 and out["micro_batches_this_rank"] == 4
    assert out["data_position"] == 63 * 32
    assert out["loss_last"] < out["loss_first"] - 1.0, (out["loss_first"], out["loss_last"])
    res2 = str(tmp_path / "r2.json")
    _worker(["--model", "resnet50", "--batch", "16", "--steps", "3", "--warmup", "2", "--global-batch", "32",
             "--result", res2])
    out2 = json.load(open(res2))
    assert out2["global_batch"] == 32 and out2["micro_batches"] == 2 and out2["loss_last"] == out2["loss_last"]


TWO_GPU_SCRIPT = """
import os, sys, json, torch, torch.distributed as dist
sys.path.insert(0, {root!r})
from trainingjob_operator_b200.runtime.worker import EngineAdapter, parse_args
rank = int(os.environ.get("RANK", "0"))
world = int(os.environ.get("WORLD_SIZE", "1"))
torch.cuda.set_device(rank)
if world > 1:
    dist.init_process_group("nccl", device_id=torch.device("cuda", rank))
args = parse_args(["--model", "gpt2-tiny", "--batch", "4", "--seq", "128", "--data", {shard!r}, "--global-batch", "12",
                   "--lr", "1e-3"])
a = EngineAdapter("gpt2-tiny", 4, 128, args)
a.bind(None)
windows, losses = [], []
for _ in range(5):
    losses.append(a.train_step())
    windows += a.samples_read
a.prepare_state()
torch.cuda.synchronize()
torch.save(a.engine.params.p32.cpu(), os.path.join({out!r}, f"p32_{{world}}_{{rank}}.pt"))
json.dump({{"rank": rank, "windows": windows, "allreduce": a.trainer.allreduce_backend, "n": a.plan.n,
            "graph": a.trainer.graph is not None or a.trainer.seg_graphs is not None, "losses": losses,
            "error": a.trainer.graph_error}}, open(os.path.join({out!r}, f"w{{world}}_{{rank}}.json"), "w"))
if world > 1:
    dist.destroy_process_group()
"""


@pytest.mark.gpu
@pytest.mark.gpu2
@pytest.mark.parametrize("allreduce", ["rs", "nccl"])
def test_two_gpus_accumulate_an_uneven_global_batch(tmp_path, allreduce):
    """k = 3 micro-batches on 2 GPUs (2 + 1), owner-sharded and bucketed NCCL: identical replicas that match one GPU
    training the same global batch, and the windows read cover [0, 5 * 12) once."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    shard = write_llmc(tmp_path / "train_000.bin", structured_corpus(200000, 1000, 999, 2))
    script = tmp_path / "acc2.py"
    script.write_text(textwrap.dedent(TWO_GPU_SCRIPT.format(root=ROOT, shard=shard, out=str(tmp_path))))
    env = dict(os.environ, AITJ_ALLREDUCE=allreduce)
    r = subprocess.run([sys.executable, str(script)], cwd=ROOT, capture_output=True, text=True, timeout=600,
                       env=dict(env, RANK="0", WORLD_SIZE="1"))
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                        "--master-addr", "127.0.0.1", "--master-port", str(_free_port()), str(script)], cwd=ROOT,
                       capture_output=True, text=True, timeout=600, env=env)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    w = [json.load(open(tmp_path / f"w2_{i}.json")) for i in range(2)]
    assert all(x["allreduce"].startswith(allreduce) and x["graph"] and not x["error"] for x in w), w
    assert [x["n"] for x in w] == [2, 1]
    assert sorted(w[0]["windows"] + w[1]["windows"]) == list(range(60))
    p = [torch.load(tmp_path / f"p32_2_{i}.pt") for i in range(2)]
    one = torch.load(tmp_path / "p32_1_0.pt")
    assert torch.equal(p[0], p[1])
    # bf16 activations, summed in a different order over the micro-batches: a bf16-rounding-sized difference after 5
    # AdamW steps at lr 1e-3 (norm of the difference against the norm of the weights)
    assert rel(p[0], one) < 2e-3, rel(p[0], one)


# ------------------------------------------------------------------------------------ 6. elastic through the control plane
@pytest.mark.slow
def test_a_job_rescaled_2_3_1_ends_where_an_unrescaled_run_ends(tmp_path):
    """``--global-batch`` on an elastic CPU job (``mlp``, gloo) submitted through ``LocalCluster`` and scaled 2 -> 3 -> 1
    while it trains: it ends at the weights of a one-rank run of the same steps, within the tolerance above."""
    from trainingjob_operator_b200.api import constants as C
    from trainingjob_operator_b200.cmd.local import LocalCluster
    from trainingjob_operator_b200.cmd.options import TrainingJobOperatorOption

    # (the rescales happen during the untimed warm-up: every rank arms the timed region at the same step)
    argv = ["--model", "mlp", "--batch", "8", "--global-batch", "48", "--steps", "10", "--warmup", "80", "--lr", "1e-2"]
    _, w_ref, _, _ = _run_recording_workers(tmp_path, 1, argv, "ref")
    out = tmp_path / "elastic"
    out.mkdir()
    script = out / "worker.py"
    script.write_text(textwrap.dedent(RECORDING_WORKER.format(root=ROOT, tests=TESTS, out=str(out))))
    worker = [sys.executable, str(script), "--cpu", "--elastic", "--step-sleep", "0.3", "--dump-outputs",
              str(out / "dump")] + argv
    job = {"apiVersion": C.API_VERSION, "kind": C.KIND, "metadata": {"name": "gb"},
           "spec": {"frameworkType": "pytorch", "replicaSpecs": {"trainer": {
               "replicas": 2, "minReplicas": 1, "maxReplicas": 3, "edlPolicy": "Manual", "restartPolicy": "Never",
               "template": {"spec": {"terminationGracePeriodSeconds": 1, "containers": [{
                   "name": "aitj-trainer", "command": worker, "workingDir": ROOT,
                   "env": [{"name": "PYTHONPATH", "value": ROOT}, {"name": "OMP_NUM_THREADS", "value": "1"}]}]}}}}}}

    def wait(fn, timeout=180.0):
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
        return json.loads(lc.jobs().get("gb").annotations.get(f"aitj.b200/{key}", "null"))

    with LocalCluster(num_gpus=0, workdir=str(tmp_path / "wd"), option=TrainingJobOperatorOption(thread_num=2)) as lc:
        try:
            lc.apply(job)
            wait(lambda: (ann(lc, "worker-trace") or {}).get("first_step_done"))
            lc.jobs().patch("gb", {"spec": {"replicaSpecs": {"trainer": {"replicas": 3}}}})
            wait(lambda: (ann(lc, "rescale-trace") or {}).get("world") == 3)
            lc.jobs().patch("gb", {"spec": {"replicaSpecs": {"trainer": {"replicas": 1}}}})
            wait(lambda: (ann(lc, "rescale-trace") or {}).get("world") == 1)
            final = lc.wait_for_phase("gb", ("Succeed", "Failed"), timeout=300)
            assert final.status.phase == "Succeed"
        finally:
            lc.jobs().delete("gb")
            time.sleep(0.5)
    steps = json.load(open(out / "steps0.json"))
    assert {s[1] for s in steps} >= {6, 3, 2}                 # rank 0 trained at W = 1, 2 and 3 (k = 6: 6, 3, 2)
    w = np.load(out / "dump" / "weights_sample.npy")
    assert float(np.linalg.norm(w - w_ref) / np.linalg.norm(w_ref)) < WEIGHT_TOL
