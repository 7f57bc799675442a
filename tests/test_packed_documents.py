"""Training on tokenized corpora with document-masked attention: the token-file loader (``runtime/data.py``), which samples
a rank reads across elastic rescales, the data position in the state hand-off and the checkpoint, the GPT-2 engine's
document mask (CPU: kernel entry points emulated, checked against the reference model), the errors for setups the mask
cannot serve, and on the GPU the masked wgmma kernels (``ops.selfcheck`` cases ``attention_docs`` / ``gpt2_docs``) and
workers training on a generated shard."""
import argparse
import json
import os
import socket
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch

import kernel_emulation as ke

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTS = os.path.dirname(os.path.abspath(__file__))


# ------------------------------------------------------------------------------------ shard writers
def write_llmc(path, tokens, magic=20240520, version=1, count=None):
    hdr = np.zeros(256, dtype="<i4")
    hdr[0], hdr[1], hdr[2] = magic, version, len(tokens) if count is None else count
    with open(path, "wb") as f:
        f.write(hdr.tobytes())
        f.write(np.asarray(tokens, dtype="<u2").tobytes())
    return str(path)


def write_raw(path, tokens):
    np.asarray(tokens, dtype="<u2").tofile(str(path))
    return str(path)


def brute_force_sample(stream_tokens, i, T, eot):
    n_win = (len(stream_tokens) - 1) // T
    w = [int(x) for x in stream_tokens[(i % n_win) * T:(i % n_win) * T + T + 1]]
    tok, tgt = w[:T], w[1:]
    ds, cur = [], 0
    for t in range(T):
        if t == 0 or tok[t] == eot:
            cur = t
        ds.append(cur)
    return tok, tgt, ds


# ------------------------------------------------------------------------------------ loader: formats
def test_llmc_and_raw_shards_round_trip(tmp_path):
    from trainingjob_operator_b200.runtime.data import TokenStream

    toks = np.random.default_rng(0).integers(0, 50257, 3000)
    for path in (write_llmc(tmp_path / "a.bin", toks), write_raw(tmp_path / "b.bin", toks)):
        s = TokenStream(path)
        assert s.n_tokens == 3000
        out = np.empty(3000, dtype=np.uint16)
        s.read(0, 3000, out)
        assert np.array_equal(out, toks)
        assert isinstance(s.shards[0], np.memmap)          # mapped, not read whole


def test_malformed_shards_raise_an_error_naming_the_file(tmp_path):
    from trainingjob_operator_b200.runtime.data import DataError, TokenStream

    toks = np.arange(100)
    bad_magic = write_llmc(tmp_path / "magic.bin", toks, magic=1234)
    with pytest.raises(DataError, match="magic.bin.*magic"):
        TokenStream(bad_magic, fmt="llmc")
    bad_version = write_llmc(tmp_path / "version.bin", toks, version=7)
    with pytest.raises(DataError, match="version.bin.*version 7"):
        TokenStream(bad_version)
    bad_size = write_llmc(tmp_path / "size.bin", toks, count=101)
    with pytest.raises(DataError, match="size.bin.*does not match"):
        TokenStream(bad_size)
    odd = tmp_path / "odd.bin"
    odd.write_bytes(b"\x01\x02\x03")
    with pytest.raises(DataError, match="odd.bin"):
        TokenStream(str(odd))
    with pytest.raises(DataError, match="no such file"):
        TokenStream(str(tmp_path / "missing_*.bin"))


def test_a_glob_of_shards_reads_as_one_stream_in_sorted_order(tmp_path):
    from trainingjob_operator_b200.runtime.data import TokenFileData

    a, b, c = np.arange(0, 150), np.arange(150, 230), np.arange(230, 400)
    write_llmc(tmp_path / "s_001.bin", b)
    write_llmc(tmp_path / "s_000.bin", a)
    write_llmc(tmp_path / "s_002.bin", c)
    d = TokenFileData(str(tmp_path / "s_*.bin"), 64, 1000, pin=False)
    assert d.stream.n_tokens == 400 and d.n_windows == (400 - 1) // 64
    for i in range(d.n_windows):
        assert np.array_equal(d.window(i), np.arange(i * 64, i * 64 + 65))   # windows 2 and 3 span shard boundaries


def test_an_out_of_range_token_raises_before_anything_is_staged(tmp_path):
    from trainingjob_operator_b200.runtime.data import DataError, TokenFileData

    toks = np.arange(1000) % 500
    toks[700] = 1000
    write_raw(tmp_path / "corpus.bin", toks)
    d = TokenFileData(str(tmp_path / "corpus.bin"), 128, 1000, pin=False)
    staged = d.stage(0, 2)
    before = [t.clone() for t in staged]
    with pytest.raises(DataError, match=r"corpus.bin: token id 1000 at token offset 700"):
        d.stage(4, 2)                   # windows 4 and 5: tokens [512, 769)
    assert all(torch.equal(t, b) for t, b in zip(staged, before))
    assert d._slots[1] is None          # the next slot was never touched


# ------------------------------------------------------------------------------------ loader: samples
def test_samples_match_a_brute_force_computation(tmp_path):
    from trainingjob_operator_b200.runtime.data import TokenFileData

    T, eot = 16, 99
    rng = np.random.default_rng(1)
    toks = rng.integers(0, 99, 16 * 6 + 1)
    toks[0] = eot                       # EOT at position 0 of window 0
    toks[20:22] = eot                   # consecutive EOTs in window 1
    toks[32:48] = rng.integers(0, 99, 16)   # window 2 holds no EOT
    toks[55] = eot
    write_llmc(tmp_path / "c.bin", toks)
    d = TokenFileData(str(tmp_path / "c.bin"), T, 100, doc_mask=True, eot=eot, pin=False)
    assert d.n_windows == 6
    tok, tgt, ds = d.stage(0, 6)
    for i in range(6):
        bt, bg, bd = brute_force_sample(toks, i, T, eot)
        assert tok[i * T:(i + 1) * T].tolist() == bt
        assert tgt[i * T:(i + 1) * T].tolist() == bg
        assert ds[i * T:(i + 1) * T].tolist() == bd
    assert tok.dtype == torch.int64 and tgt.dtype == torch.int64 and ds.dtype == torch.int32
    assert ds[16:32].tolist()[3:7] == [0, 4, 5, 5]      # window 1: EOTs at positions 4 and 5
    assert ds[32:48].tolist() == [0] * 16
    # wrap-around: sample 6 + i is sample i of the next epoch
    again = d.stage(6, 6)               # (the other staging slot: the first one still holds samples 0..5)
    assert all(torch.equal(a, b) for a, b in zip(again, (tok, tgt, ds)))
    assert all(np.array_equal(a, b) for a, b in zip(d.sample(1), d.sample(13)))


# ------------------------------------------------------------------------------------ which samples a rank reads
class _StubTrainer:
    def __init__(self, world, rank):
        self.world, self.rank, self.step_count = world, rank, 0

    def step(self, *host):
        self.step_count += 1
        return 0.0


def _adapter_on(data, batch, world, rank, position):
    from trainingjob_operator_b200.runtime.worker import EngineAdapter

    a = EngineAdapter.__new__(EngineAdapter)
    a.data, a.batch, a.data_position = data, batch, position
    a.trainer = _StubTrainer(world, rank)
    return a


def test_ranks_read_disjoint_consecutive_samples_and_rescales_leave_no_gap(tmp_path):
    from trainingjob_operator_b200.runtime.data import TokenFileData

    write_raw(tmp_path / "c.bin", np.arange(20000) % 1000)
    B = 3
    pos = 0
    seen = []
    for world, steps in ((2, 3), (3, 2), (1, 4)):
        for _ in range(steps):
            per_rank = []
            for r in range(world):
                d = TokenFileData(str(tmp_path / "c.bin"), 32, 1000, pin=False)
                a = _adapter_on(d, B, world, r, pos)
                a.train_step()
                per_rank.append(d.samples_read)
                new_pos = a.data_position
            assert new_pos == pos + world * B
            flat = [i for rr in per_rank for i in rr]
            assert flat == list(range(pos, pos + world * B))   # rank r: [pos + r*B, pos + (r+1)*B)
            seen += flat
            pos = new_pos
    assert seen == list(range(len(seen))) and len(seen) == B * (2 * 3 + 3 * 2 + 1 * 4)


# ------------------------------------------------------------------------------------ data position hand-off / checkpoint
SYNC_SCRIPT = """
import os, sys, json, torch, torch.distributed as dist
sys.path.insert(0, {root!r})
from trainingjob_operator_b200.runtime.rendezvous import sync_state
rank = int(os.environ["RANK"])
dist.init_process_group("gloo", rank=rank, world_size=2)

class WithPosition:
    def __init__(self, steps, pos):
        self.step_count, self.data_position, self.w = steps, pos, torch.full((4,), float(rank))
    def state_tensors(self):
        return [self.w]
    def after_state_load(self):
        pass

class WithoutPosition(WithPosition):
    def __init__(self, steps):
        super().__init__(steps, 0)
        del self.data_position

a = WithPosition(steps=5 + 3 * rank, pos=100 + 50 * rank)      # rank 1 holds more optimizer steps: the source
loop = sync_state(a, 10 + rank, torch.device("cpu"))
b = WithoutPosition(steps=9 - rank)                              # rank 0 is the source here
loop_b = sync_state(b, 20 + rank, torch.device("cpu"))
print("RESULT " + json.dumps({{"rank": rank, "pos": a.data_position, "steps": a.step_count, "loop": loop,
      "w": a.w.tolist(), "b_has_pos": hasattr(b, "data_position"), "b_loop": loop_b, "b_w": b.w.tolist()}}), flush=True)
dist.destroy_process_group()
"""


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def test_sync_state_hands_the_data_position_from_the_elected_source(tmp_path):
    script = tmp_path / "sync.py"
    script.write_text(textwrap.dedent(SYNC_SCRIPT.format(root=ROOT)))
    port = _free_port()
    procs = [subprocess.Popen([sys.executable, str(script)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                              env=dict(os.environ, RANK=str(r), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port),
                                       OMP_NUM_THREADS="1")) for r in range(2)]
    res = []
    for p in procs:
        out = p.communicate(timeout=120)[0]
        assert p.returncode == 0, out[-3000:]
        res.append(json.loads(next(ln for ln in out.splitlines() if ln.startswith("RESULT "))[7:]))
    for r in res:
        assert r["pos"] == 150 and r["steps"] == 8 and r["loop"] == 11 and r["w"] == [1.0] * 4
        assert r["b_has_pos"] is False and r["b_loop"] == 20 and r["b_w"] == [0.0] * 4


def test_a_checkpoint_round_trip_restores_the_data_position(tmp_path):
    from trainingjob_operator_b200.runtime import worker as W

    class A:
        def __init__(self, pos):
            self.data_position, self.t = pos, torch.arange(8, dtype=torch.float32) * (pos + 1)

        def state_tensors(self):
            return [self.t]

        def after_state_load(self):
            pass

    args = argparse.Namespace(ckpt_dir=str(tmp_path / "ck"))
    W.save_checkpoint(args, A(1234), 17)
    W.checkpointer(args).wait()
    b = A(0)
    assert W.load_checkpoint(args, b) == 17
    assert b.data_position == 1234 and torch.equal(b.t, torch.arange(8, dtype=torch.float32) * 1235)


# ------------------------------------------------------------------------------------ engine in emulation
def install_doc_attention(monkeypatch=None):
    """``kernel_emulation.install``: its attention entry points also take the document mask."""
    ke.install(monkeypatch)


def _doc_batch(B, T, vocab, eot, seed):
    g = torch.Generator().manual_seed(seed)
    tok = torch.randint(0, vocab - 1, (B, T), generator=g)
    tok[tok == eot] = 0
    for b, starts in enumerate(([5, 6, 70, 127], [64, 65])[:B]):
        tok[b, starts] = eot
    from trainingjob_operator_b200.runtime.data import doc_starts

    ds = torch.from_numpy(doc_starts(tok.numpy(), eot))
    return tok, torch.roll(tok, -1, dims=1), ds


def test_gpt2_engine_with_document_mask_matches_the_reference_model(monkeypatch):
    from trainingjob_operator_b200.models.gpt2 import GPT2Config, GPT2Engine, GPT2Reference

    install_doc_attention(monkeypatch)
    cfg = GPT2Config(vocab_size=1000, n_layer=2, n_head=4, n_embd=256, block_size=128, name="t")
    B, T = 2, 128
    eng = GPT2Engine(cfg, B, T, "cpu", seed=3, gemm_backend="wgmma", doc_mask=True)
    assert eng.attn_impl == "wgmma" and eng.attn_bwd_impl == "wgmma"
    assert [t.dtype for t in eng.input_tensors()] == [torch.int64, torch.int64, torch.int32]
    g = torch.Generator().manual_seed(9)
    for s_ in eng.params.specs:
        if len(s_.shape) == 1:
            eng.params.w32(s_.name).add_(torch.randn(s_.shape, generator=g) * 0.05)
    eng.params.refresh_compute_copy()
    ref = GPT2Reference(cfg, eng.params)
    tok, tgt, ds = _doc_batch(B, T, cfg.vocab_size, 999, 5)
    for dst, src in zip(eng.input_tensors(), (tok, tgt, ds)):
        dst.copy_(src.reshape(-1))
    eng.params.g32.zero_()
    eng.forward()
    eng.backward()
    loss = ref(tok, tgt, ds)
    loss.backward()
    assert abs(float(eng.loss) - float(loss.detach())) < 2e-2 * float(loss.detach())
    for name in ("wte", "wpe", "h0.qkv_w", "h0.qkv_b", "h0.proj_w", "h0.proj_b", "h0.fc_w", "h0.fc_b", "h0.fc2_w",
                 "h0.fc2_b", "h0.ln1_w", "h0.ln1_b", "h1.ln2_w", "h1.ln2_b", "h1.fc2_w", "h1.qkv_w", "lnf_w", "lnf_b"):
        got, want = eng.params.grad(name), ref.p(name).grad
        assert float((got - want).norm() / (want.norm() + 1e-12)) < 6e-2, name
    # the mask matters: the unmasked reference differs
    assert abs(float(GPT2Reference(cfg, eng.params)(tok, tgt).detach()) - float(loss.detach())) > 1e-4


def test_document_mask_is_refused_where_the_wgmma_attention_cannot_run(monkeypatch):
    from trainingjob_operator_b200.models.bert import BertConfig, BertEngine
    from trainingjob_operator_b200.models.gpt2 import GPT2Config, GPT2Engine

    install_doc_attention(monkeypatch)
    cfg = GPT2Config(vocab_size=1000, n_layer=1, n_head=4, n_embd=256, block_size=256, name="t")
    with pytest.raises(ValueError, match="gemm_backend is 'cublas'"):
        GPT2Engine(cfg, 2, 128, "cpu", gemm_backend="cublas", doc_mask=True)
    with pytest.raises(ValueError, match="192 is not a multiple of 128"):
        GPT2Engine(cfg, 2, 192, "cpu", doc_mask=True)
    with pytest.raises(ValueError, match="head dim 128"):
        GPT2Engine(GPT2Config(vocab_size=1000, n_layer=1, n_head=2, n_embd=256, block_size=128), 2, 128, "cpu",
                   doc_mask=True)
    with pytest.raises(ValueError, match="needs causal attention"):       # BERT's bidirectional attention
        GPT2Engine(cfg, 2, 128, "cpu", causal=False, doc_mask=True)
    bert = BertEngine(BertConfig.tiny(), 2, 128, "cpu")
    assert bert.doc_mask is False and len(bert.input_tensors()) == 3
    with pytest.raises(ValueError, match="needs causal"):
        from trainingjob_operator_b200.ops import functional as F

        F._check_doc_start(torch.zeros(256, dtype=torch.int32), 2, 128, causal=False)
    from trainingjob_operator_b200.ops import functional as F

    with pytest.raises(ValueError, match="int32"):
        F._check_doc_start(torch.zeros(256, dtype=torch.int64), 2, 128, causal=True)


def test_worker_rejects_data_flags_it_cannot_serve():
    from trainingjob_operator_b200.runtime.worker import parse_args

    with pytest.raises(SystemExit):
        parse_args(["--model", "gpt2-tiny", "--doc-mask"])
    with pytest.raises(SystemExit):
        parse_args(["--model", "bert", "--data", "x.bin"])
    with pytest.raises(SystemExit):
        parse_args(["--model", "gpt2-tiny", "--data", "x.bin", "--doc-mask"])          # 50256 >= 1000
    a = parse_args(["--model", "gpt2-tiny", "--data", "x.bin", "--doc-mask", "--eot-token", "999"])
    assert a.doc_mask and a.eot_token == 999 and a.data == "x.bin"
    a = parse_args(["--model", "gpt2"])
    assert a.data == "" and not a.doc_mask and a.eot_token == 50256


# ------------------------------------------------------------------------------------ worker loop in emulation
WORKER_SCRIPT = """
import os, sys
sys.path.insert(0, {root!r}); sys.path.insert(0, {tests!r})
import test_packed_documents as tpd
tpd.install_doc_attention()
from trainingjob_operator_b200.runtime import worker as W
W.build_adapter = lambda args, device: W.EngineAdapter(args.model, args.batch, args.seq, args, device="cpu")
sys.exit(W.main(sys.argv[1:]))
"""


def structured_corpus(n_tokens, vocab, eot, seed):
    """Documents that are runs of consecutive ids from a random start, each opened by ``eot``: learnable structure."""
    rng = np.random.default_rng(seed)
    out = []
    while len(out) < n_tokens:
        n = int(rng.integers(8, 200))
        start = int(rng.integers(0, vocab - 1))
        out += [eot] + [(start + i) % (vocab - 1) for i in range(n)]
    return np.asarray(out[:n_tokens])


def _run_cpu_workers(tmp_path, n, argv, env_extra=None):
    script = tmp_path / "worker_docs.py"
    script.write_text(textwrap.dedent(WORKER_SCRIPT.format(root=ROOT, tests=TESTS)))
    port = _free_port()
    procs = []
    for r in range(n):
        env = dict(os.environ, RANK=str(r), WORLD_SIZE=str(n), LOCAL_RANK=str(r), MASTER_ADDR="127.0.0.1",
                   MASTER_PORT=str(port), OMP_NUM_THREADS="2", AITJ_WORKDIR=str(tmp_path), TRAININGJOB_NAME="docs",
                   AITJ_CKPT_ASYNC="0", **(env_extra or {}))
        env.pop("AITJ_MASTER", None)
        res = tmp_path / f"result{r}.json"
        procs.append((res, subprocess.Popen([sys.executable, str(script), "--cpu", "--result", str(res)] + argv, env=env,
                                            stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    out = []
    for res, p in procs:
        log = p.communicate(timeout=600)[0]
        assert p.returncode == 0, log[-4000:]
        out.append((json.load(open(res)) if res.exists() else None, log))
    return out


@pytest.mark.slow
def test_two_rank_worker_trains_on_a_shard_with_document_mask_and_resumes_the_data_position(tmp_path):
    shard = write_llmc(tmp_path / "train_000.bin", structured_corpus(40000, 1000, 999, 0))
    argv = ["--model", "gpt2-tiny", "--batch", "2", "--seq", "128", "--steps", "4", "--warmup", "3", "--ckpt-every", "2",
            "--ckpt-dir", str(tmp_path / "ck"), "--data", shard, "--doc-mask", "--eot-token", "999"]
    res = _run_cpu_workers(tmp_path, 2, argv)
    r0, log0 = res[0]
    assert r0 and r0["world"] == 2 and r0["steps_done"] == 7, (r0, log0[-2000:])
    assert r0["data_position"] == 7 * 2 * 2 and r0["describe"]["doc_mask"] is True
    assert r0["h2d_bytes_per_step"] == 2 * 128 * 20
    assert r0["loss_last"] < r0["loss_first"]
    res2 = _run_cpu_workers(tmp_path, 2, argv, {"TRAININGJOB_REPLICA_RESTARTCOUNT": "1"})
    r0b, log0b = res2[0]
    assert "resumed from checkpoint at step 6, data position 24" in log0b, log0b[-2000:]
    assert r0b["steps_done"] == 7 and r0b["data_position"] == 28


# ------------------------------------------------------------------------------------ GPU
def _run_case(name: str, timeout: int = 420):
    r = subprocess.run([sys.executable, "-m", "trainingjob_operator_b200.ops.selfcheck", "--case", name], cwd=ROOT,
                       capture_output=True, text=True, timeout=timeout)
    sys.stdout.write(r.stdout[-4000:])
    sys.stderr.write(r.stderr[-2000:])
    assert r.returncode == 0, f"selfcheck {name} failed:\n{r.stdout[-3000:]}\n{r.stderr[-1500:]}"


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["attention_docs", "gpt2_docs"])
def test_document_masked_kernels_and_engine(case):
    _run_case(case)


@pytest.mark.gpu
def test_worker_trains_gpt2_tiny_on_a_shard_with_document_mask(tmp_path):
    """One GPU, through the worker: a CUDA graph, a finite loss, and on documents of consecutive ids the loss falls well
    below ln(vocab)."""
    shard = write_llmc(tmp_path / "train_000.bin", structured_corpus(400000, 1000, 999, 0))
    res = str(tmp_path / "r.json")
    env = dict(os.environ, WORLD_SIZE="1", RANK="0", PYTHONPATH=ROOT)
    env.pop("AITJ_MASTER", None)
    r = subprocess.run([sys.executable, "-m", "trainingjob_operator_b200.runtime.worker", "--model", "gpt2-tiny", "--batch",
                        "16", "--seq", "128", "--steps", "150", "--warmup", "3", "--lr", "1e-3", "--data", shard,
                        "--doc-mask", "--eot-token", "999", "--result", res], cwd=ROOT, env=env, capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    out = json.load(open(res))
    print(json.dumps({k: out[k] for k in ("loss_first", "loss_last", "ms_per_step", "data_position")}))
    assert out["cuda_graph"] and out["loss_last"] == out["loss_last"]
    assert out["data_position"] == 153 * 16
    assert out["loss_last"] < 0.5 * np.log(1000), out["loss_last"]


@pytest.mark.gpu
def test_document_masked_job_through_the_control_plane(tmp_path):
    from trainingjob_operator_b200.cmd.local import LocalCluster

    shard = write_llmc(tmp_path / "train_000.bin", structured_corpus(100000, 1000, 999, 1))
    worker = [sys.executable, "-m", "trainingjob_operator_b200.runtime.worker", "--model", "gpt2-tiny", "--batch", "4",
              "--seq", "128", "--steps", "5", "--warmup", "3", "--data", shard, "--doc-mask", "--eot-token", "999"]
    job = {"apiVersion": "elasticdeeplearning.ai/v1", "kind": "AITrainingJob", "metadata": {"name": "docs-e2e"},
           "spec": {"frameworkType": "pytorch", "replicaSpecs": {"trainer": {"replicas": 1, "template": {"spec": {
               "containers": [{"name": "aitj-trainer", "command": worker, "workingDir": ROOT,
                               "env": [{"name": "PYTHONPATH", "value": ROOT}],
                               "resources": {"limits": {"nvidia.com/gpu": 1}}}]}}}}}}
    with LocalCluster(num_gpus=1, workdir=str(tmp_path)) as lc:
        lc.apply(job)
        final = lc.wait_for_phase("docs-e2e", ("Succeed", "Failed"), timeout=300)
        logs = ""
        if final.status.phase != "Succeed":
            for fn in os.listdir(os.path.join(lc.workdir, "logs")):
                logs += open(os.path.join(lc.workdir, "logs", fn)).read()[-2000:]
        assert final.status.phase == "Succeed", logs
        m = json.loads(final.annotations["aitj.b200/metrics"])
        assert m["samples_per_sec"] > 0 and m["cuda_graph"] and m["loss_last"] == m["loss_last"]


RS_SCRIPT = """
import os, sys, json, argparse, torch, torch.distributed as dist
sys.path.insert(0, {root!r})
from trainingjob_operator_b200.runtime.worker import EngineAdapter, parse_args
rank = int(os.environ["RANK"])
torch.cuda.set_device(rank)
dist.init_process_group("nccl", device_id=torch.device("cuda", rank))
args = parse_args(["--model", "gpt2-tiny", "--batch", "4", "--seq", "128", "--data", {shard!r}, "--doc-mask",
                   "--eot-token", "999"])
a = EngineAdapter("gpt2-tiny", 4, 128, args)
a.bind(None)
windows = []
for _ in range(4):
    loss = a.train_step()
    windows += a.data.samples_read
json.dump({{"rank": rank, "windows": windows, "allreduce": a.trainer.allreduce_backend, "loss": loss}},
          open(os.path.join({out!r}, f"windows{{rank}}.json"), "w"))
dist.destroy_process_group()
"""


@pytest.mark.gpu
@pytest.mark.gpu2
def test_two_ranks_on_the_owner_sharded_path_read_disjoint_windows(tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    shard = write_llmc(tmp_path / "train_000.bin", structured_corpus(100000, 1000, 999, 2))
    script = tmp_path / "rs.py"
    script.write_text(textwrap.dedent(RS_SCRIPT.format(root=ROOT, shard=shard, out=str(tmp_path))))
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                        "--master-addr", "127.0.0.1", "--master-port", str(_free_port()), str(script)], cwd=ROOT,
                       capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    w = [json.load(open(tmp_path / f"windows{i}.json")) for i in range(2)]
    assert all(x["allreduce"].startswith("rs") for x in w), w
    assert not set(w[0]["windows"]) & set(w[1]["windows"])
    assert sorted(w[0]["windows"] + w[1]["windows"]) == list(range(32))
