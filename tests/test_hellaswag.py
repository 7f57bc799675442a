"""HellaSwag scoring of GPT-2 workers (``--hellaswag``): llm.c's eval file, the packing of completions as documents
(``runtime/hellaswag.py``), the kernels ``embedding_doc_fwd`` / ``choice_score`` (``ops/csrc/hellaswag.cu``),
``GPT2Engine.score_forward``, the worker's schedule and reports, and ``cmd/hellaswag``.

CPU tests run the engine with the kernel entry points emulated: ``tests/kernel_emulation.py`` plus the stand-ins of the
two HellaSwag entry points below, which apply the wrappers' own checks.  GPU tests run the hand-written kernels on an
H100."""
import io
import json
import os
import socket
import subprocess
import sys
import textwrap
import types

import numpy as np
import pytest
import torch

import kernel_emulation as ke
from test_packed_documents import structured_corpus, write_llmc
from trainingjob_operator_b200.ops import functional as F
from trainingjob_operator_b200.runtime.data import DataError

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTS = os.path.dirname(os.path.abspath(__file__))


# ------------------------------------------------------------------------------------ stand-ins
def embedding_doc_fwd(tok, wte, wpe, doc_start, out, T):
    M, _C = F.check_embedding_doc_fwd(tok, wte, wpe, doc_start, out, T)
    pos = torch.arange(M, device=tok.device) % T - doc_start.long()
    out.copy_(wte[tok].float() + wpe[pos].float())
    return out


def choice_score(loss, spans, labels, mean, acc):
    E = F.check_choice_score(loss, spans, labels, mean, acc)
    sp = spans.long().tolist()
    m = torch.tensor([[float(loss[a:a + n].double().sum()) / n for a, n in row] for row in sp], dtype=torch.float64)
    mean.copy_(m.float())
    pick = [min(range(4), key=lambda c, r=r: (float(mean[r, c]), c)) for r in range(E)]
    acc[0] += float(sum(int(p == int(l)) for p, l in zip(pick, labels.tolist())))
    acc[1] += float(E)
    return mean


def install_hellaswag(monkeypatch=None):
    """``kernel_emulation.install`` and the two HellaSwag entry points."""
    ke.install(monkeypatch)
    for name, fn in (("embedding_doc_fwd", embedding_doc_fwd), ("choice_score", choice_score)):
        if monkeypatch is not None:
            monkeypatch.setattr(F, name, fn)
        else:
            setattr(F, name, fn)


# ------------------------------------------------------------------------------------ llm.c's format, written here
def llmc_stream(examples, overrides=None):
    """The uint16 stream and header of llm.c's ``write_evalfile`` for ``examples`` ((label, ctx, [endings])).
    ``overrides``: {example: {field index: value}} to write a malformed stream."""
    stream, longest = [], 0
    for i, (label, ctx, ends) in enumerate(examples):
        ex = [65535, 0, i, label, len(ends), len(ctx)] + list(ctx)
        for e in ends:
            ex += [len(e)] + list(e)
        ex[1] = 2 * len(ex)
        for k, v in (overrides or {}).get(i, {}).items():
            ex[k] = v
        longest = max(longest, ex[1])
        stream += ex
    head = np.zeros(256, dtype="<i4")
    head[:4] = (20240522, 1, len(examples), longest)
    return head, np.asarray(stream, dtype="<u2")


def write_file(path, examples, overrides=None, header=None, cut=0):
    head, stream = llmc_stream(examples, overrides)
    for k, v in (header or {}).items():
        head[k] = v
    blob = head.tobytes() + stream.tobytes()
    with open(path, "wb") as f:
        f.write(blob[:len(blob) - cut])
    return str(path)


def random_examples(rng, n, vocab, ctx=(1, 40), end=(1, 12)):
    out = []
    for _ in range(n):
        c = rng.integers(0, vocab, int(rng.integers(ctx[0], ctx[1] + 1))).tolist()
        ends = [rng.integers(0, vocab, int(rng.integers(end[0], end[1] + 1))).tolist() for _ in range(4)]
        out.append((int(rng.integers(0, 4)), c, ends))
    return out


# ------------------------------------------------------------------------------------ 1. reader
def test_the_reader_reads_back_what_llmc_writes(tmp_path):
    from trainingjob_operator_b200.runtime.hellaswag import read_examples, write_examples

    exs = random_examples(np.random.default_rng(0), 30, 1000)
    path = write_file(tmp_path / "hs.bin", exs)
    got = read_examples(path, 1000, 128)
    assert [g.index for g in got] == list(range(30))
    for g, (label, ctx, ends) in zip(got, exs):
        assert g.label == label and g.ctx.tolist() == ctx and [e.tolist() for e in g.ends] == ends
    # the package's writer (fixtures, benchmark) writes the same bytes
    assert open(write_examples(str(tmp_path / "pkg.bin"), exs), "rb").read() == open(path, "rb").read()


def _bad_files():
    ok = [(1, [5, 6, 7], [[1], [2, 3], [4], [5]]), (2, [8, 9], [[1, 2], [3], [4], [5, 6, 7]]),
          (0, [3], [[9], [8], [7], [6]])]
    long_ctx = [(0, list(range(100)), [[1] * 30, [2], [3], [4]])]
    return [
        ("magic", ok, dict(header={0: 20240520}), "magic 20240520", None),
        ("version", ok, dict(header={1: 2}), "version 2", None),
        ("delimiter", ok, dict(overrides={1: {0: 65534}}), "missing start delimiter", 1),
        ("byte count", ok, dict(overrides={1: {1: 26}}), "byte count 26 does not match", 1),
        ("count low", ok, dict(header={2: 2}), "counts 2 examples, the file holds more", None),
        ("count high", ok, dict(header={2: 4}), "counts 4 examples, the file holds 3", None),
        ("truncated", ok, dict(cut=4), "truncated file", 2),
        ("completions", ok, dict(overrides={1: {4: 3}}), "3 completions, not 4", 1),
        ("label", ok, dict(overrides={2: {3: 4}}), "label 4 is not below 4", 2),
        ("empty context", [(0, [], [[1], [2], [3], [4]])], {}, "empty context", 0),
        ("empty ending", [(0, [1], [[1], [], [3], [4]])], {}, "ending 1 is empty", 0),
        ("vocabulary", [ok[0], (0, [5, 1000], [[1], [2], [3], [4]])], {}, "token id 1000 is outside", 1),
        ("too long", long_ctx, {}, "completion 0 takes 129 input positions, more than --seq 128", 0),
    ]


@pytest.mark.parametrize("case", _bad_files(), ids=lambda c: c[0])
def test_the_reader_refuses_malformed_files(tmp_path, case):
    from trainingjob_operator_b200.runtime.hellaswag import read_examples

    _name, exs, kw, what, example = case
    path = write_file(tmp_path / "bad.bin", exs, **kw)
    with pytest.raises(DataError) as e:
        read_examples(path, 1000, 128)
    msg = str(e.value)
    assert what in msg and path in msg, msg
    if example is not None:
        assert f"example {example}:" in msg, msg


# ------------------------------------------------------------------------------------ 2. packer
@pytest.mark.parametrize("B,T,seed", [(4, 128, 0), (8, 256, 1), (5, 384, 2), (16, 1024, 3)])
def test_the_packer_keeps_its_invariants(tmp_path, B, T, seed):
    from trainingjob_operator_b200.runtime.hellaswag import HellaSwagData, read_examples

    rng = np.random.default_rng(seed)
    exs = random_examples(rng, 300, 1000, ctx=(1, T // 3), end=(1, T // 4))
    path = write_file(tmp_path / "hs.bin", exs)
    d = HellaSwagData(path, 1000, B, T)
    ref = read_examples(path, 1000, T)
    K, M = d.micro_batches, B * T
    assert d.first[0] == 0 and d.first[-1] == len(exs) == d.examples and len(d.first) == K + 1
    assert d.tok.shape == (K, M) and d.doc_start.dtype == torch.int32
    filled = 0
    for k in range(K):
        tok, tgt, ds, spans, labels = (t.numpy() for t in d.inputs(k))
        owner = np.full(M, -1)
        want_tgt = np.full(M, -1)
        prev_end = None
        for j, ex in enumerate(ref[d.first[k]:d.first[k + 1]]):
            assert labels[j] == ex.label
            for c, end in enumerate(ex.ends):
                first, n = spans[j, c]
                n_ctx = len(ex.ctx)
                a, L = first - (n_ctx - 1), n_ctx + len(end) - 1
                assert n == len(end) and 0 <= a and a + L <= M
                assert a // T == (a + L - 1) // T, "a completion straddles two rows"
                assert (owner[a:a + L] == -1).all(), "two completions overlap"
                owner[a:a + L] = 1
                seq = np.concatenate([ex.ctx, end])
                assert (tok[a:a + L] == seq[:-1]).all() and (ds[a:a + L] == a % T).all()
                want_tgt[first:first + n] = end
                # placement: right after the previous completion, or at the start of the next row when it does not fit
                if prev_end is not None:
                    if prev_end % T + L <= T and prev_end % T != 0:
                        assert a == prev_end, (k, j, c)
                    else:
                        assert a == -(-prev_end // T) * T, (k, j, c)
                prev_end = a + L
                filled += L
        if k + 1 < K:
            # the next micro-batch's first example would not have fitted after the last one of this
            nxt = ref[d.first[k + 1]]
            r, p = divmod(prev_end, T)
            for end in nxt.ends:
                L = len(nxt.ctx) + len(end) - 1
                if p + L > T:
                    r, p = r + 1, 0
                p += L
            assert r >= B or (r == B - 1 and p > T)
        pad = owner == -1
        assert (tgt == want_tgt).all(), "targets >= 0 exactly at the ending-predicting positions"
        assert (tok[pad] == 0).all() and (ds[pad] == np.arange(M)[pad] % T).all()
        rows = ds.reshape(B, T)
        assert (rows[:, 0] == 0).all() and (np.diff(rows, axis=1) >= 0).all()
        assert (rows <= np.arange(T)).all()
    assert abs(d.fill - filled / (K * M)) < 1e-12
    # the plan depends on nothing but the file, B and T: every world size covers every micro-batch once
    for W in (1, 2, 3, 7):
        got = sorted(m for r in range(W) for m in d.plan(W, r))
        assert got == list(range(K)) and d.plan(W, 0) == tuple(range(0, K, W))


def test_an_example_that_fits_no_micro_batch_is_refused(tmp_path):
    from trainingjob_operator_b200.runtime.hellaswag import HellaSwagData

    path = write_file(tmp_path / "hs.bin", [(0, list(range(60)), [[1] * 60, [2] * 60, [3] * 60, [4] * 60])])
    with pytest.raises(DataError, match=r"hs\.bin: example 0: .* do not fit in a micro-batch of 2 rows of 128"):
        HellaSwagData(path, 1000, 2, 128)


# ------------------------------------------------------------------------------------ 3. emulated engine
def _tiny_cfg():
    from trainingjob_operator_b200.models.gpt2 import GPT2Config

    return GPT2Config(vocab_size=1000, n_layer=2, n_head=4, n_embd=256, block_size=128, name="t")


def _shared_context_examples(rng, n, vocab):
    """Examples whose completions share a long context and end in one or two tokens: a completion that saw its
    neighbour's tokens, or positions counted from the row's start, would score differently."""
    out = []
    for _ in range(n):
        ctx = rng.integers(0, vocab, int(rng.integers(10, 30))).tolist()
        ends = [rng.integers(0, vocab, int(rng.integers(1, 3))).tolist() for _ in range(4)]
        out.append((int(rng.integers(0, 4)), ctx, ends))
    return out


def _reference_means(ref, examples):
    """Per-completion mean NLL of the fp32 model, each completion alone in a row from position 0."""
    out = []
    dev = ref.p("wte").device
    with torch.no_grad():
        for ex in examples:
            row = []
            for end in ex.ends:
                seq = torch.from_numpy(np.concatenate([ex.ctx, end])).to(dev)
                tok = seq[:-1].view(1, -1)
                tgt = torch.full_like(tok, -100)
                tgt[0, len(ex.ctx) - 1:] = seq[len(ex.ctx):]
                row.append(float(ref(tok, tgt)))
            out.append(row)
    return np.asarray(out)


def _score_emulated(monkeypatch, tmp_path, B=4, T=128, n=14):
    from trainingjob_operator_b200.models.gpt2 import GPT2Engine, GPT2Reference
    from trainingjob_operator_b200.runtime.hellaswag import HellaSwagData, read_examples

    install_hellaswag(monkeypatch)
    cfg = _tiny_cfg()
    eng = GPT2Engine(cfg, B, T, "cpu", seed=3)
    with torch.no_grad():
        # an opinionated model: larger token embeddings give wide margins between the completions, larger position
        # embeddings make every position count, and sharper attention makes a token of another document count
        P = eng.params
        P.w32("wte")[:cfg.vocab_size].mul_(6.0)
        P.w32("wpe").mul_(30.0)
        for i in range(cfg.n_layer):
            P.w32(f"h{i}.qkv_w").mul_(5.0)
        P.refresh_compute_copy()
    path = write_file(tmp_path / "hs.bin", _shared_context_examples(np.random.default_rng(11), n, cfg.vocab_size))
    data = HellaSwagData(path, cfg.vocab_size, B, T)
    assert data.micro_batches >= 2
    ref = GPT2Reference(cfg, eng.params)
    return eng, data, read_examples(path, cfg.vocab_size, T), ref


def _engine_means(eng, data):
    means = []
    eng.choice_acc.zero_()
    for k in range(data.micro_batches):
        tok, tgt, ds, spans, labels = data.inputs(k)
        eng.tok.copy_(tok)
        eng.tgt.copy_(tgt)
        means.append(eng.score_forward(ds, spans, labels, spans.shape[0]).clone())
    return torch.cat(means).double().numpy()


TINY_TOL = 5e-2    # bf16 activations of the engine against the fp32 model (as for eval_forward at this size)


def test_packed_scores_match_the_fp32_model_one_completion_per_row(monkeypatch, tmp_path):
    eng, data, exs, ref = _score_emulated(monkeypatch, tmp_path)
    P = eng.params
    before = [t.clone() for t in (P.p32, P.m, P.v, P.g32, P.p16, eng.eval_acc)]
    got = _engine_means(eng, data)
    assert all(torch.equal(x, y) for x, y in zip(before, (P.p32, P.m, P.v, P.g32, P.p16, eng.eval_acc)))
    want = _reference_means(ref, exs)
    err = np.abs(got - want).max()
    assert err < TINY_TOL, err
    srt = np.sort(want, 1)
    assert (srt[:, 1] - srt[:, 0] > 2 * TINY_TOL).all(), "the fixture needs clear margins"
    labels = np.array([e.label for e in exs])
    ref_correct = int((want.argmin(1) == labels).sum())
    assert float(eng.choice_acc[1]) == len(exs) and int(eng.choice_acc[0]) == ref_correct
    assert (got.argmin(1) == want.argmin(1)).all()


def test_the_comparison_fails_without_document_positions_or_the_document_mask(monkeypatch, tmp_path):
    """Mutations: positions counted from the row's start (embedding_fwd's), or the attention without the document mask.
    Either moves the scores well past the tolerance and changes some answers."""
    eng, data, exs, ref = _score_emulated(monkeypatch, tmp_path)
    want = _reference_means(ref, exs)
    T = eng.T

    def row_positions(tok, wte, wpe, doc_start, out, T_):
        return ke.embedding_fwd(tok, wte, wpe, out, T_)

    monkeypatch.setattr(F, "embedding_doc_fwd", row_positions)
    bad = _engine_means(eng, data)
    assert np.abs(bad - want).max() > 10 * TINY_TOL and (bad.argmin(1) != want.argmin(1)).any()
    monkeypatch.setattr(F, "embedding_doc_fwd", embedding_doc_fwd)
    attn = F.attention_fwd

    def unmasked(qkv, out, lse, B, T_, H, causal=True, scale=0.0, doc_start=None):
        return attn(qkv, out, lse, B, T_, H, causal=causal, scale=scale)

    monkeypatch.setattr(F, "attention_fwd", unmasked)
    bad = _engine_means(eng, data)
    assert T == 128 and np.abs(bad - want).max() > 10 * TINY_TOL and (bad.argmin(1) != want.argmin(1)).any()


def test_score_forward_refuses_what_the_kernels_cannot_serve(monkeypatch):
    from trainingjob_operator_b200.models.gpt2 import GPT2Config, GPT2Engine

    install_hellaswag(monkeypatch)
    sp, lab, ds = torch.zeros(1, 4, 2, dtype=torch.int32), torch.zeros(1, dtype=torch.int32), torch.zeros(256,
                                                                                                        dtype=torch.int32)
    for kw, cfg, T, what in ((dict(gemm_backend="cublas"), _tiny_cfg(), 128, "gemm_backend is 'cublas'"),
                             ({}, _tiny_cfg(), 64, "sequence length 64 is not a multiple of 128"),
                             ({}, GPT2Config(vocab_size=1000, n_layer=1, n_head=2, n_embd=256, block_size=128), 128,
                              "head dim 128 is not 64")):
        eng = GPT2Engine(cfg, 2, T, "cpu", seed=0, **kw)
        with pytest.raises(ValueError, match=what):
            eng.score_forward(ds[:2 * T], sp, lab, 1)


def test_the_wrappers_check_every_argument():
    bf = torch.bfloat16
    tok, wte, wpe = torch.zeros(256, dtype=torch.int64), torch.zeros(100, 64, dtype=bf), torch.zeros(128, 64, dtype=bf)
    ds, out = torch.zeros(256, dtype=torch.int32), torch.zeros(256, 64, dtype=bf)
    assert F.check_embedding_doc_fwd(tok, wte, wpe, ds, out, 128) == (256, 64)
    for bad, what in ((dict(doc_start=ds.long()), "doc_start must be torch.int32"),
                      (dict(doc_start=torch.zeros(258, dtype=torch.int32)[1:257]), "doc_start must be 8-byte aligned"),
                      (dict(doc_start=ds[:128]), "doc_start must hold 256"), (dict(T=100), "not a multiple of T"),
                      (dict(T=256), r"T 256 must be in \[1, 128\]"), (dict(out=out[:, :32]), "out must be contiguous"),
                      (dict(tok=tok.int()), "tok must be torch.int64"),
                      (dict(wpe=torch.zeros(128, 72, dtype=bf)), "same width")):
        a = dict(tok=tok, wte=wte, wpe=wpe, doc_start=ds, out=out, T=128)
        a.update(bad)
        with pytest.raises(ValueError, match=what):
            F.embedding_doc_fwd(**a)
    loss, sp, lab = torch.zeros(256), torch.zeros(3, 4, 2, dtype=torch.int32), torch.zeros(3, dtype=torch.int32)
    mean, acc = torch.zeros(3, 4), torch.zeros(2, dtype=torch.float64)
    assert F.check_choice_score(loss, sp, lab, mean, acc) == 3
    for bad, what in ((dict(spans=sp[:0]), "E >= 1"), (dict(spans=sp.view(3, 8)), "spans must have 3 dimensions"),
                      (dict(spans=torch.zeros(3, 2, 2, dtype=torch.int32)), r"spans must be \[E, 4, 2\]"),
                      (dict(labels=lab.long()), "labels must be torch.int32"), (dict(labels=lab[:2]), "labels must hold 3"),
                      (dict(mean=torch.zeros(3, 5)), r"mean must be \[3, 4\]"), (dict(acc=acc.float()), "acc must be"),
                      (dict(loss=loss.double()), "loss must be torch.float32")):
        a = dict(loss=loss, spans=sp, labels=lab, mean=mean, acc=acc)
        a.update(bad)
        with pytest.raises(ValueError, match=what):
            F.choice_score(**a)


# ------------------------------------------------------------------------------------ 4. workers over gloo
WORKER = """
import os, sys, json, atexit
sys.path.insert(0, {root!r}); sys.path.insert(0, {tests!r})
import test_hellaswag as th
th.install_hellaswag()
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
                   MASTER_PORT=str(port), OMP_NUM_THREADS="1", AITJ_WORKDIR=str(out), TRAININGJOB_NAME="hs",
                   AITJ_CKPT_ASYNC="0")
        env.pop("AITJ_MASTER", None)
        procs.append(subprocess.Popen([sys.executable, str(script), "--cpu", "--result", str(out / "result.json"),
                                       "--dump-outputs", str(out / "dump"), "--ckpt-dir", str(out / "ckpt")] + argv,
                                      env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True))
    logs = [p.communicate(timeout=900)[0] for p in procs]
    for p, log in zip(procs, logs):
        assert p.returncode == 0, log[-4000:]
    steps = [json.load(open(out / f"steps{r}.json")) for r in range(n)]
    return json.load(open(out / "result.json")), np.load(out / "dump" / "weights_sample.npy"), steps, logs[0], out


@pytest.mark.slow
def test_scoring_changes_no_training_step_and_is_the_same_at_any_world_size(monkeypatch, tmp_path):
    """Two ranks, --global-batch 8 in micro-batches of 2, 4 steps, --hellaswag-every 2: the same training losses and
    final weights, bit for bit, as without scoring; the same (correct, examples) as one rank at every scored step; and
    cmd/hellaswag on the last checkpoint prints the last record."""
    train = write_llmc(tmp_path / "train_000.bin", structured_corpus(60000, 1000, 999, 3))
    hs = write_file(tmp_path / "hs.bin", random_examples(np.random.default_rng(5), 40, 1000, ctx=(5, 40), end=(1, 15)))
    base = ["--model", "gpt2-tiny", "--batch", "2", "--seq", "128", "--steps", "3", "--warmup", "1", "--lr", "1e-3",
            "--data", train, "--global-batch", "8"]
    sc = ["--hellaswag", hs, "--hellaswag-every", "2", "--ckpt-every", "4"]
    r2, w2, s2, log, _ = _run_workers(tmp_path, 2, base + sc, "w2hs")
    r2n, w2n, s2n, _, _ = _run_workers(tmp_path, 2, base, "w2")
    r1, _, _, _, out1 = _run_workers(tmp_path, 1, base + sc, "w1hs")
    assert s2 == s2n and np.array_equal(w2, w2n)
    assert "hellaswag" not in r2n and "hellaswag_acc_last" not in r2n
    assert [h["step"] for h in r2["hellaswag"]] == [2, 4]
    assert all(h["examples"] == 40 and h["acc"] == h["correct"] / 40 and h["ms"] >= 0 for h in r2["hellaswag"])
    assert r2["hellaswag_acc_last"] == r2["hellaswag"][-1]["acc"]
    assert [(h["correct"], h["examples"]) for h in r2["hellaswag"]] == \
        [(h["correct"], h["examples"]) for h in r1["hellaswag"]]
    assert "step 4: hellaswag acc" in log
    # the checkpoint of step 4 (one rank's job), scored by the command with the worker's --batch and --seq
    install_hellaswag(monkeypatch)
    from trainingjob_operator_b200.cmd import hellaswag as cmd

    buf = io.StringIO()
    assert cmd.main(["--cpu", "--model", "gpt2-tiny", "--ckpt", str(out1 / "ckpt" / "hs.pt"), "--data", hs,
                     "--batch", "2", "--seq", "128"], out=buf) == 0
    rec = json.loads(buf.getvalue())
    last = r1["hellaswag"][-1]
    assert (rec["correct"], rec["examples"], rec["acc"]) == (last["correct"], last["examples"], last["acc"])


# ------------------------------------------------------------------------------------ 5. arguments and reports
def test_the_worker_refuses_scoring_it_cannot_run(monkeypatch, tmp_path):
    from trainingjob_operator_b200.runtime.worker import EngineAdapter, parse_args

    for argv, what in ((["--model", "bert-tiny", "--hellaswag", "x.bin"], "GPT-2 models only"),
                       (["--model", "gpt2-tiny", "--gemm", "cublas", "--hellaswag", "x.bin"], "--gemm wgmma"),
                       (["--model", "gpt2-tiny", "--seq", "200", "--hellaswag", "x.bin"], "--seq a multiple of 128"),
                       (["--model", "gpt2-tiny", "--hellaswag-every", "5"], "--hellaswag-every needs --hellaswag"),
                       (["--model", "gpt2-tiny", "--hellaswag", "x.bin", "--hellaswag-every", "-1"], "cannot be negative")):
        err = io.StringIO()
        monkeypatch.setattr(sys, "stderr", err)
        with pytest.raises(SystemExit):
            parse_args(argv)
        assert what in err.getvalue(), err.getvalue()
    monkeypatch.undo()
    args = parse_args(["--model", "gpt2-tiny", "--seq", "128"])
    assert args.hellaswag == "" and args.hellaswag_every == 0
    install_hellaswag(monkeypatch)
    bad = write_file(tmp_path / "hs_bad.bin", [(0, [1], [[1], [2], [3], [4]])], header={0: 1})
    with pytest.raises(DataError, match=r"hs_bad\.bin: magic 1"):
        EngineAdapter("gpt2-tiny", 2, 128, parse_args(["--model", "gpt2-tiny", "--seq", "128", "--hellaswag", bad]),
                      device="cpu")


def _job(name, metrics):
    st = types.SimpleNamespace(phase="Running", rendezvous=None)
    return types.SimpleNamespace(name=name, status=st, annotations={"aitj.b200/metrics": json.dumps(metrics)})


def test_hellaswag_reaches_top_the_job_gauge_and_the_final_report():
    from trainingjob_operator_b200.cli.kubectl import CLI
    from trainingjob_operator_b200.controller.trainingjob import observe_worker_reports
    from trainingjob_operator_b200.runtime.elastic import ElasticWatcher
    from trainingjob_operator_b200.utils import metrics

    jobs = [_job("with-hs", {"samples_per_sec": 100.0, "steps_done": 8, "hellaswag_acc": 0.2875, "hellaswag_step": 8,
                             "eval_loss": 3.25}),
            _job("no-hs", {"samples_per_sec": 50.0})]
    lister = types.SimpleNamespace(list=lambda: types.SimpleNamespace(items=jobs))
    cs = types.SimpleNamespace(elasticdeeplearning_v1=lambda: types.SimpleNamespace(aitrainingjobs=lambda ns: lister))
    out = io.StringIO()
    cli = CLI.__new__(CLI)
    cli.cs, cli.out = cs, out
    cli.p = lambda s="": out.write(s + "\n")
    assert cli.top("default", False) == 0
    lines = out.getvalue().splitlines()
    assert lines[0].split()[-3:] == ["HELLASWAG", "EVAL", "LOSS"]
    assert lines[1].split()[-2:] == ["0.2875", "3.2500"] and lines[2].split()[-2:] == ["<none>", "<none>"]

    metrics.reset()
    base = {"metadata": {"namespace": "default", "name": "j", "annotations": {}}}
    cur = {"metadata": {"namespace": "default", "name": "j", "annotations": {
        "aitj.b200/metrics": json.dumps({"samples_per_sec": 10.0, "hellaswag_acc": 0.3, "hellaswag_step": 4})}}}
    observe_worker_reports(base, cur)
    assert 'aitj_job_hellaswag_acc{job="j",namespace="default"} 0.3' in metrics.render()
    metrics.reset()

    w = ElasticWatcher.__new__(ElasticWatcher)
    sent = {}
    w._annotate = lambda k, v: sent.update({k: v})
    w.report_result({"samples_per_sec": 1.0, "hellaswag": [{"step": 2, "acc": 0.25}, {"step": 4, "acc": 0.5}]})
    m = sent["aitj.b200/metrics"]
    assert m["hellaswag_acc"] == 0.5 and m["hellaswag_step"] == 4
    w.report_result({"samples_per_sec": 1.0})
    assert "hellaswag_acc" not in sent["aitj.b200/metrics"]


def test_the_example_manifest_scores_hellaswag():
    import yaml

    doc = yaml.safe_load(open(os.path.join(ROOT, "examples", "gpt2-hellaswag.yaml")))
    argv = doc["spec"]["replicaSpecs"]["trainer"]["template"]["spec"]["containers"][0]["args"]
    assert "--hellaswag" in argv and "--hellaswag-every" in argv
    from trainingjob_operator_b200.runtime.worker import parse_args

    args = parse_args(argv[argv.index("trainingjob_operator_b200.runtime.worker") + 1:])
    assert args.hellaswag and args.hellaswag_every > 0 and args.seq % 128 == 0


# ------------------------------------------------------------------------------------ GPU
def _doc_starts(B, T, rng):
    """Random packed rows: documents of 1 to 300 positions, doc_start non-decreasing, 0 at each row start."""
    ds = np.zeros((B, T), dtype=np.int32)
    for b in range(B):
        p = 0
        while p < T:
            n = int(rng.integers(1, 300))
            ds[b, p:p + n] = p
            p += n
    return torch.from_numpy(ds.reshape(-1))


@pytest.mark.gpu
@pytest.mark.parametrize("C", [768, 1024, 1280, 1600])
def test_embedding_doc_fwd_is_a_gather_bit_for_bit(C):
    g = torch.Generator(device="cuda").manual_seed(C)
    B, T, V = 8, 1024, 50304
    wte = torch.randn(V, C, device="cuda", generator=g).bfloat16()
    wpe = torch.randn(1024, C, device="cuda", generator=g).bfloat16()
    tok = torch.randint(0, V, (B * T,), device="cuda", generator=g)
    ds = _doc_starts(B, T, np.random.default_rng(C)).cuda()
    out = torch.full((B * T + 2, C), 7.0, device="cuda", dtype=torch.bfloat16)
    F.embedding_doc_fwd(tok, wte, wpe, ds, out[1:-1], T)
    pos = torch.arange(B * T, device="cuda") % T - ds.long()
    want = (wte[tok].float() + wpe[pos].float()).bfloat16()
    torch.cuda.synchronize()
    assert torch.equal(out[1:-1], want)
    assert bool((out[0] == 7).all() and (out[-1] == 7).all())


def _run_choice_score(loss, spans, labels):
    E = spans.shape[0]
    mean = torch.full((E + 2, 4), float("nan"), device="cuda")
    mean[0] = mean[-1] = 123.0
    acc = torch.full((4,), -5.0, device="cuda", dtype=torch.float64)
    acc[1:3] = 0
    F.choice_score(loss, spans, labels, mean[1:-1], acc[1:3])
    torch.cuda.synchronize()
    assert bool((mean[0] == 123).all() and (mean[-1] == 123).all()), "a sentinel row was written"
    assert float(acc[0]) == -5.0 and float(acc[3]) == -5.0
    return mean[1:-1].cpu(), acc[1:3].cpu()


@pytest.mark.gpu
def test_choice_score_against_fp64():
    rng = np.random.default_rng(0)
    B, T = 16, 1024
    M = B * T
    loss = torch.from_numpy(rng.gamma(2.0, 2.0, M).astype(np.float32))
    E = 3001
    n = rng.integers(1, 200, (E, 4))
    n[0] = (1, T, 1, T)                      # spans of length 1 and T
    n[1] = (T, T, 1, 5)
    first = rng.integers(0, M - n + 1)
    spans = np.stack([first, n], 2).astype(np.int32)
    # exact ties: completions over the same positions, the tied pair at every place in the example
    for e, (a, b) in zip(range(2, 14), [(0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3)] * 2):
        spans[e, b] = spans[e, a]
    labels = rng.integers(0, 4, E).astype(np.int32)
    want = np.array([[loss[a:a + k].double().sum().item() / k for a, k in row] for row in spans])
    mean, acc = _run_choice_score(loss.cuda(), torch.from_numpy(spans).cuda(), torch.from_numpy(labels).cuda())
    assert not torch.isnan(mean).any()
    rel = np.abs(mean.double().numpy() - want) / want
    assert rel.max() < 2 ** -23, rel.max()   # the fp64 sum, rounded once to fp32
    m32 = mean.numpy()
    pick = np.array([min(range(4), key=lambda c, r=r: (m32[r, c], c)) for r in range(E)])
    assert float(acc[1]) == E and float(acc[0]) == float((pick == labels).sum())
    srt = np.sort(want, 1)
    clear = srt[:, 1] - srt[:, 0] > 1e-5 * srt[:, 0]
    assert (pick[clear] == want.argmin(1)[clear]).all()
    # the first of a tied pair wins: all right with the label on the first, none with the label on the second
    ties = spans[2:14]
    tie_pairs = [(0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3)] * 2
    lowest = want[2:14].min(1)
    rows = [e for e, (a, b) in zip(range(12), tie_pairs) if want[2 + e, a] == lowest[e]]
    assert rows, "no tied pair holds the lowest mean; change the seed"
    sub = torch.from_numpy(ties[rows]).cuda()
    first_lab = torch.tensor([tie_pairs[e][0] for e in rows], dtype=torch.int32, device="cuda")
    second_lab = torch.tensor([tie_pairs[e][1] for e in rows], dtype=torch.int32, device="cuda")
    assert float(_run_choice_score(loss.cuda(), sub, first_lab)[1][0]) == len(rows)
    assert float(_run_choice_score(loss.cuda(), sub, second_lab)[1][0]) == 0


def _gpu_file(tmp_path, vocab, n, seed):
    rng = np.random.default_rng(seed)
    return write_file(tmp_path / "hs.bin", random_examples(rng, n, vocab, ctx=(8, 90), end=(2, 30)))


def _gpu_reference_check(tmp_path, cfg, B, T, n_examples):
    """score_forward on the packed file against the fp32 model one completion per row, and the tolerance derived from
    the existing evaluation path: the engine's eval_forward (training attention, positions from 0) on the same
    completions placed one per row, held to the same model."""
    from trainingjob_operator_b200.models.gpt2 import GPT2Engine, GPT2Reference
    from trainingjob_operator_b200.runtime.hellaswag import HellaSwagData, read_examples

    path = _gpu_file(tmp_path, cfg.vocab_size, n_examples, 1)
    data = HellaSwagData(path, cfg.vocab_size, B, T, pin=True)
    exs = read_examples(path, cfg.vocab_size, T)
    eng = GPT2Engine(cfg, B, T, "cuda", seed=7)
    got = []
    eng.choice_acc.zero_()
    for k in range(data.micro_batches):
        tok, tgt, ds, spans, labels = data.inputs(k)
        eng.tok.copy_(tok)
        eng.tgt.copy_(tgt)
        got.append(eng.score_forward(ds, spans.cuda(), labels.cuda(), spans.shape[0]).double().cpu())
    got = torch.cat(got).numpy()
    correct = int(eng.choice_acc[0])
    # the reference, each completion alone in a row of its length; eval_forward, one completion per row
    want = _reference_means(GPT2Reference(cfg, eng.params).cuda(), exs)
    flat = [(e, c) for e in range(len(exs)) for c in range(4)]
    base = np.zeros((len(exs), 4))
    for i in range(0, len(flat), B):
        chunk = flat[i:i + B]
        tok = torch.zeros(B, T, dtype=torch.int64)
        tgt = torch.full((B, T), -1, dtype=torch.int64)
        for r, (e, c) in enumerate(chunk):
            ex = exs[e]
            seq = torch.from_numpy(np.concatenate([ex.ctx, ex.ends[c]]))
            tok[r, :len(seq) - 1] = seq[:-1]
            tgt[r, len(ex.ctx) - 1:len(seq) - 1] = seq[len(ex.ctx):]
        eng.tok.copy_(tok.view(-1))
        eng.tgt.copy_(tgt.view(-1))
        eng.eval_acc.zero_()
        eng.eval_forward()
        ev = eng.losses.view(B, T).double().cpu()
        for r, (e, c) in enumerate(chunk):
            base[e, c] = float(ev[r][tgt[r] >= 0].mean())
    eval_err = np.abs(base - want).max()
    tol = 2 * eval_err + 2e-3
    err = np.abs(got - want).max()
    print(f"score_forward vs fp32: max |d| {err:.2e}; eval_forward vs fp32 {eval_err:.2e}; tol 2 x that + 2e-3 = "
          f"{tol:.2e}; {data.micro_batches} micro-batches, fill {data.fill:.3f}")
    assert err <= tol, (err, tol)
    srt = np.sort(want, 1)
    clear = srt[:, 1] - srt[:, 0] > 2 * err
    assert (got.argmin(1)[clear] == want.argmin(1)[clear]).all()
    labels = np.array([e.label for e in exs])
    assert int(eng.choice_acc[1]) == len(exs) and correct == int((got.argmin(1) == labels).sum())


@pytest.mark.gpu
def test_gpt2_small_score_forward_against_the_fp32_model(tmp_path):
    from trainingjob_operator_b200.models.gpt2 import GPT2Config

    _gpu_reference_check(tmp_path, GPT2Config.small(), 4, 1024, 120)


@pytest.mark.gpu
def test_a_wide_engine_score_forward_against_the_fp32_model(tmp_path):
    from trainingjob_operator_b200.models.gpt2 import GPT2Config

    _gpu_reference_check(tmp_path, GPT2Config(n_layer=2, n_head=25, n_embd=1600, name="xl-2"), 4, 1024, 60)


@pytest.mark.gpu
def test_scoring_under_a_captured_training_graph_changes_no_training_step(tmp_path):
    """cuDNN attention (the default) in a captured training graph; scoring between two steps runs the wgmma attention
    under the document mask on the same layer buffers.  From the same saved state, the next step is run twice without
    scoring and once after it: its loss is bit for bit the same, and its weights differ from the first run by at most
    twice what the two runs without scoring differ by (the weight-gradient, bias and LayerNorm reductions add with
    atomics, in an order that changes from run to run; where the repeat is bitwise, so must the scored run be)."""
    from trainingjob_operator_b200.models.gpt2 import GPT2Config, GPT2Engine
    from trainingjob_operator_b200.runtime.hellaswag import HellaSwagData
    from trainingjob_operator_b200.runtime.trainer import EngineTrainer

    assert os.environ.get("AITJ_ATTN", "cudnn") == "cudnn"
    cfg = GPT2Config(n_layer=4)
    B, T = 4, 1024
    eng = GPT2Engine(cfg, B, T, "cuda", seed=1)
    assert eng.attn_impl == "cudnn"
    tr = EngineTrainer(eng)
    g = torch.Generator().manual_seed(0)
    batches = [(torch.randint(0, 50257, (B * T,), generator=g).pin_memory(),
                torch.randint(0, 50257, (B * T,), generator=g).pin_memory()) for _ in range(3)]
    for b in batches[:2]:
        tr.step(*b)
    assert tr.graph is not None
    P = eng.params
    saved = [t.clone() for t in P.state_tensors()]
    step0 = tr.step_count
    data = HellaSwagData(_gpu_file(tmp_path, cfg.vocab_size, 40, 2), cfg.vocab_size, B, T, pin=True)

    def next_step(score):
        for t, s in zip(P.state_tensors(), saved):
            t.copy_(s)
        P.refresh_compute_copy()
        tr.step_count = step0
        if score:
            correct, examples = tr.score(data.inputs(k) for k in range(data.micro_batches))
            assert examples == 40 and 0 <= correct <= 40
        loss = tr.step(*batches[2])
        torch.cuda.synchronize()
        return loss, P.p32.clone()

    (loss_a, w_a), (loss_a2, w_a2), (loss_b, w_b) = next_step(False), next_step(False), next_step(True)
    assert loss_a == loss_a2 == loss_b, (loss_a, loss_a2, loss_b)
    spread = float((w_a2 - w_a).abs().max())
    d = float((w_b - w_a).abs().max())
    print(f"weights after the step: scored vs unscored max |d| {d:.3e}, unscored run-to-run {spread:.3e}")
    assert d <= 2 * spread, (d, spread)


def _worker(argv, timeout=900):
    env = dict(os.environ, WORLD_SIZE="1", RANK="0", PYTHONPATH=ROOT)
    env.pop("AITJ_MASTER", None)
    r = subprocess.run([sys.executable, "-m", "trainingjob_operator_b200.runtime.worker"] + argv, cwd=ROOT, env=env,
                       capture_output=True, text=True, timeout=timeout)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    return r.stdout


@pytest.mark.gpu
def test_one_gpu_worker_scores_hellaswag(tmp_path):
    from trainingjob_operator_b200.runtime.elastic import ElasticWatcher

    train = write_llmc(tmp_path / "train_000.bin", structured_corpus(400000, 1000, 999, 0))
    hs = write_file(tmp_path / "hs.bin", random_examples(np.random.default_rng(3), 200, 1000, ctx=(5, 60), end=(1, 20)))
    res = str(tmp_path / "r.json")
    log = _worker(["--model", "gpt2-tiny", "--batch", "8", "--seq", "128", "--steps", "40", "--warmup", "3", "--lr",
                   "1e-3", "--data", train, "--hellaswag", hs, "--hellaswag-every", "20", "--result", res])
    out = json.load(open(res))
    print(json.dumps({k: out[k] for k in ("loss_first", "loss_last", "ms_per_step", "hellaswag")}))
    assert [h["step"] for h in out["hellaswag"]] == [20, 40, 43]
    assert all(h["examples"] == 200 and 0 <= h["correct"] <= 200 for h in out["hellaswag"])
    assert out["hellaswag_acc_last"] == out["hellaswag"][-1]["acc"]
    assert out["cuda_graph"] and not out["graph_error"] and "hellaswag acc" in log
    w = ElasticWatcher.__new__(ElasticWatcher)
    sent = {}
    w._annotate = lambda k, v: sent.update({k: v})
    w.report_result(out)
    assert sent["aitj.b200/metrics"]["hellaswag_acc"] == out["hellaswag"][-1]["acc"]


TWO_GPU_SCRIPT = """
import os, sys, json, torch, torch.distributed as dist
sys.path.insert(0, {root!r})
from trainingjob_operator_b200.runtime.worker import EngineAdapter, parse_args
rank = int(os.environ.get("RANK", "0"))
world = int(os.environ.get("WORLD_SIZE", "1"))
torch.cuda.set_device(rank)
if world > 1:
    dist.init_process_group("nccl", device_id=torch.device("cuda", rank))
args = parse_args(["--model", "gpt2", "--batch", "4", "--seq", "1024", "--hellaswag", {hs!r}])
a = EngineAdapter("gpt2", 4, 1024, args)
a.bind(None)
json.dump(a.score(), open(os.path.join({out!r}, f"w{{world}}_{{rank}}.json"), "w"))
if world > 1:
    dist.destroy_process_group()
"""


@pytest.mark.gpu
@pytest.mark.gpu2
def test_two_gpus_score_as_one(tmp_path):
    """GPT-2 small: packing and per-row compute do not depend on the world size, so two GPUs give exactly the same
    (correct, examples) as one."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    hs = _gpu_file(tmp_path, 50257, 300, 4)
    script = tmp_path / "hs2.py"
    script.write_text(TWO_GPU_SCRIPT.format(root=ROOT, hs=hs, out=str(tmp_path)))
    for world in (1, 2):
        port = _free_port()
        procs = [subprocess.Popen([sys.executable, str(script)], cwd=ROOT, stdout=subprocess.PIPE,
                                  stderr=subprocess.STDOUT, text=True,
                                  env=dict(os.environ, RANK=str(r), WORLD_SIZE=str(world), MASTER_ADDR="127.0.0.1",
                                           MASTER_PORT=str(port)))
                 for r in range(world)]
        logs = [p.communicate(timeout=900)[0] for p in procs]
        assert all(p.returncode == 0 for p in procs), "\n".join(l[-3000:] for l in logs)
    one = json.load(open(tmp_path / "w1_0.json"))
    for r in range(2):
        two = json.load(open(tmp_path / f"w2_{r}.json"))
        assert (two["correct"], two["examples"]) == (one["correct"], one["examples"]) and one["examples"] == 300
