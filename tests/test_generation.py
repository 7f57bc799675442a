"""Text generation from GPT-2 workers (``--generate-every``) and checkpoints (``cmd/generate.py``): the decode kernels
(``ops/csrc/decode.cu``: ``attention_decode``, ``embedding_decode``, ``sample_tokens``), ``models.generate.GPT2Generator``,
the worker's flags, schedule and results, and the llm.c tokenizer.

CPU tests run the engine with the kernel entry points emulated (``tests/kernel_emulation.py`` for the training kernels,
the plain-PyTorch stand-ins below for the decode kernels, which apply the wrappers' own argument checks) and gloo
between processes; the GPU tests run the hand-written kernels on an H100."""
import io
import json
import os
import struct
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch

import kernel_emulation as ke
from test_heldout_eval import _free_port, install_xent
from test_packed_documents import structured_corpus, write_llmc
from trainingjob_operator_b200.ops import functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTS = os.path.dirname(os.path.abspath(__file__))


# ------------------------------------------------------------------------------------ stand-ins of the decode kernels
def philox_first_word(seed: int, seq: int, pos: int) -> int:
    """Philox4x32-10 of counter (pos, seq, 0, 0) and key (seed low, seed high): the first output word, as the kernel."""
    m = 0xFFFFFFFF
    c0, c1, c2, c3 = pos & m, seq & m, 0, 0
    k0, k1 = seed & m, (seed >> 32) & m
    for _ in range(10):
        p0, p1 = 0xD2511F53 * c0, 0xCD9E8D57 * c2
        c0, c1, c2, c3 = ((p1 >> 32) ^ c1 ^ k0) & m, p1 & m, ((p0 >> 32) ^ c3 ^ k1) & m, p0 & m
        k0, k1 = (k0 + 0x9E3779B9) & m, (k1 + 0xBB67AE85) & m
    return c0


def attention_decode(qkv, cache, pos, out, part, H):
    S, Tmax = F.check_attention_decode(qkv, cache, pos, out, part, H)
    p, C = int(pos[0]), H * 64
    cache[:, p, 0].copy_(qkv[:, C:2 * C].view(S, H, 64))
    cache[:, p, 1].copy_(qkv[:, 2 * C:].view(S, H, 64))
    q = qkv[:, :C].float().view(S, H, 64)
    k, v = cache[:, :p + 1, 0].float(), cache[:, :p + 1, 1].float()
    w = torch.softmax(torch.einsum("shd,sthd->sht", q, k) * 0.125, -1)
    out.copy_(torch.einsum("sht,sthd->shd", w, v).reshape(S, C))
    return out


def embedding_decode(tok, wte, wpe, pos, out):
    F.check_embedding_decode(tok, wte, wpe, pos, out)
    out.copy_(wte[tok].float() + wpe[int(pos[0])].float())
    return out


def sample_tokens(logits, vocab, tok, out_tokens, prompt, prompt_len, pos, temperature, top_k, seed, first_seq=0):
    S = F.check_sample_tokens(logits, vocab, tok, out_tokens, prompt, prompt_len, pos, temperature, top_k, seed,
                              first_seq)
    p = int(pos[0])
    for s in range(S):
        if p + 1 < prompt_len:
            t = int(prompt[s, p + 1])
        else:
            z = logits[s, :vocab].double()
            if temperature == 0 or top_k == 1:
                t = int(torch.argmax(z))                      # the first of equal maxima
            else:
                keep = z >= torch.topk(z, top_k).values[-1] if 0 < top_k < vocab else torch.ones_like(z, dtype=bool)
                w = torch.exp((z - z.max()) / temperature) * keep
                u = (philox_first_word(seed, first_seq + s, p) >> 8) / float(1 << 24)
                c = torch.cumsum(w, 0)
                hit = torch.nonzero(c > u * float(c[-1]))
                t = int(hit[0]) if hit.numel() else int(torch.nonzero(keep)[-1])
        tok[s] = t
        if p + 1 < out_tokens.shape[1]:
            out_tokens[s, p + 1] = t
    pos[0] = p + 1
    return tok


def install_decode(monkeypatch=None):
    """The training kernels' stand-ins (``kernel_emulation.install``), the cross-entropy ones and the decode ones."""
    ke.install(monkeypatch)
    install_xent(monkeypatch)
    for name, fn in (("attention_decode", attention_decode), ("embedding_decode", embedding_decode),
                     ("sample_tokens", sample_tokens)):
        if monkeypatch is not None:
            monkeypatch.setattr(F, name, fn)
        else:
            setattr(F, name, fn)


def _cfg():
    from trainingjob_operator_b200.models.gpt2 import GPT2Config

    return GPT2Config(vocab_size=1000, n_layer=2, n_head=4, n_embd=256, block_size=128, name="t")


def _engine(monkeypatch, B=2, T=64, seed=3):
    from trainingjob_operator_b200.models.gpt2 import GPT2Engine

    install_decode(monkeypatch)
    return GPT2Engine(_cfg(), B, T, "cpu", seed=seed)


def _forward_logits(eng, tok):
    """The training forward's logits rows (``GPT2Engine.forward`` before its loss turns them into dlogits)."""
    eng.tok.copy_(tok.reshape(-1))
    eng._trunk()
    eng._linear(eng.lnf, eng.params.w16("wte"), eng.logits)
    return eng.logits[:, :eng.cfg.vocab_size].float().view(tok.shape[0], tok.shape[1], -1)


# ------------------------------------------------------------------------------------ 1. teacher forcing
def test_teacher_forced_decode_gives_the_training_forwards_logits(monkeypatch):
    from trainingjob_operator_b200.models.generate import GPT2Generator

    eng = _engine(monkeypatch)
    B, T = eng.B, eng.T
    tok = torch.randint(0, 1000, (B, T), generator=torch.Generator().manual_seed(1))
    want = _forward_logits(eng, tok)
    before = [t.clone() for t in (eng.params.p32, eng.params.p16, eng.params.g32, eng.logits, eng.tok)]
    gen = GPT2Generator(eng, B, T + 1)
    got = torch.empty(B, T, 1000)
    out = gen.generate(tok, 1, temperature=0.0, logits_out=got)
    assert torch.equal(out[:, :T], tok)                              # the prompt is forced at every position
    err = float((got - want).abs().max())
    assert err < 3e-2 * float(want.abs().max()), err                  # bf16 activations on both sides
    after = (eng.params.p32, eng.params.p16, eng.params.g32, eng.logits, eng.tok)
    assert all(torch.equal(x, y) for x, y in zip(before, after)), "generation touched the engine's state"
    assert int(out[0, T]) == int(torch.argmax(got[0, T - 1]))


# ------------------------------------------------------------------------------------ 2. greedy against re-forwards
def _reference_logits(ref, tok):
    """Last-position logits of the fp32 reference model over the prefix ``tok`` [S, t]."""
    import torch.nn.functional as TF

    seen = {}
    ce = TF.cross_entropy

    def grab(z, t):
        seen["z"] = z
        return ce(z, t)

    TF.cross_entropy = grab
    try:
        with torch.no_grad():
            ref(tok, torch.zeros_like(tok))
    finally:
        TF.cross_entropy = ce
    return seen["z"].view(tok.shape[0], tok.shape[1], -1)[:, -1]


def test_greedy_generation_is_argmax_over_full_reforwards(monkeypatch):
    from trainingjob_operator_b200.models.generate import GPT2Generator
    from trainingjob_operator_b200.models.gpt2 import GPT2Reference

    eng = _engine(monkeypatch, seed=11)
    with torch.no_grad():                             # sharper logits than at initialisation: clear margins
        eng.params.w32("wte").mul_(25.0)
        eng.params.refresh_compute_copy()
    ref = GPT2Reference(eng.cfg, eng.params)
    prompt = [5, 17, 400]
    out = GPT2Generator(eng, 2, 24).generate(prompt, 20, temperature=0.0)
    seq = torch.tensor([prompt, prompt])
    for i in range(20):
        z = _reference_logits(ref, seq)
        top2 = torch.topk(z, 2, dim=-1).values
        assert float((top2[:, 0] - top2[:, 1]).min()) > 0.05 * float(z.abs().max()), "margins too small to compare"
        seq = torch.cat([seq, torch.argmax(z, -1, keepdim=True)], 1)
    assert torch.equal(out, seq)


# ------------------------------------------------------------------------------------ 3. keying of the draws
def test_a_sequence_draws_the_same_tokens_alone_or_with_others(monkeypatch):
    from trainingjob_operator_b200.models.generate import GPT2Generator, generation_seed

    eng = _engine(monkeypatch)
    prompt = [999, 3]
    five = GPT2Generator(eng, 5, 20).generate(prompt, 18, temperature=1.0, top_k=50, seed=7)
    one = GPT2Generator(eng, 1, 20)
    for i in range(5):
        assert torch.equal(one.generate(prompt, 18, temperature=1.0, top_k=50, seed=7, first_seq=i)[0], five[i])
    assert not all(torch.equal(five[0], five[i]) for i in range(1, 5))
    other = GPT2Generator(eng, 5, 20).generate(prompt, 18, temperature=1.0, top_k=50, seed=8)
    assert not torch.equal(other, five)
    assert generation_seed(0, 2) != generation_seed(0, 4) and generation_seed(0, 2) != generation_seed(1, 2)
    assert generation_seed(0, 2) == generation_seed(0, 2)


def test_top_k_and_vocab_bound_the_draws(monkeypatch):
    install_decode(monkeypatch)
    S, Vp, V, k = 64, 1024, 1000, 5
    logits = torch.randn(S, Vp, generator=torch.Generator().manual_seed(0)).bfloat16()
    logits[:, V:] = 100.0                                # padding columns are never drawn, however large
    tok, out = torch.zeros(S, dtype=torch.int64), torch.zeros(S, 4, dtype=torch.int64)
    prompt, pos = torch.zeros(S, 1, dtype=torch.int64), torch.zeros(2, dtype=torch.int32)
    F.sample_tokens(logits, V, tok, out, prompt, 1, pos, 2.0, k, 123)
    top = torch.topk(logits[:, :V].float(), k, -1).indices
    assert all(int(tok[s]) in top[s].tolist() for s in range(S)) and int(pos[0]) == 1
    assert torch.equal(out[:, 1], tok)


# ------------------------------------------------------------------------------------ 4. workers over gloo
WORKER = """
import os, sys, json, time, atexit
sys.path.insert(0, {root!r}); sys.path.insert(0, {tests!r})
import test_generation as tg
tg.install_decode()
from trainingjob_operator_b200.ops import lib
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
    if hasattr(ad, "generator"):
        generate = ad.generate
        def slow(*a, **k):
            # a generation that is slow and launches much: the step figures must not see either
            time.sleep(1.5)
            lib.LAUNCHES += 100000
            return generate(*a, **k)
        ad.generate = slow
    return ad
W.build_adapter = build
atexit.register(lambda: json.dump(RECORD, open(os.path.join({out!r}, "steps%s.json" % os.environ["RANK"]), "w")))
sys.exit(W.main(sys.argv[1:]))
"""


def _run_workers(tmp_path, n, argv, tag):
    out = tmp_path / tag
    out.mkdir()
    script = out / "worker.py"
    script.write_text(textwrap.dedent(WORKER.format(root=ROOT, tests=TESTS, out=str(out))))
    port = _free_port()
    procs = []
    for r in range(n):
        env = dict(os.environ, RANK=str(r), WORLD_SIZE=str(n), LOCAL_RANK=str(r), MASTER_ADDR="127.0.0.1",
                   MASTER_PORT=str(port), OMP_NUM_THREADS="1", AITJ_WORKDIR=str(out), TRAININGJOB_NAME="gen",
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


def _tokenizer_file(path, n, version=2, eot=None, magic=20240328, truncate=0):
    hdr = [0] * 256
    hdr[0], hdr[1], hdr[2] = magic, version, n
    if version == 2:
        hdr[3] = n - 1 if eot is None else eot
    body = b"".join(bytes([len(t)]) + t for t in (_token_bytes(i) for i in range(n)))
    data = struct.pack("<256I", *hdr) + body
    with open(path, "wb") as f:
        f.write(data[:len(data) - truncate])
    return str(path)


def _token_bytes(i):
    return "é".encode() if i == 7 else f"<{i}>".encode()


@pytest.mark.slow
def test_generation_changes_no_training_step_and_is_the_same_at_any_world_size(tmp_path, monkeypatch):
    """Two ranks, 1 + 4 steps, --generate-every 2: generations before step 2 and 4 and after step 5, the same on one
    rank; the same losses and final weights, bit for bit, as without generation; neither the generation's time nor its
    launches reach the step figures.  The checkpoint of the last step gives the last generation's tokens through
    cmd/generate.py."""
    train = write_llmc(tmp_path / "train_000.bin", structured_corpus(60000, 1000, 999, 3))
    tk = _tokenizer_file(tmp_path / "tok.bin", 1000)
    base = ["--model", "gpt2-tiny", "--batch", "2", "--seq", "128", "--steps", "4", "--warmup", "1", "--lr", "1e-3",
            "--data", train, "--eot-token", "999", "--ckpt-every", "5", "--global-batch", "4"]
    gen = ["--generate-every", "2", "--generate-count", "3", "--generate-tokens", "6", "--top-k", "40",
           "--temperature", "0.9", "--tokenizer", tk]
    r2, w2, s2, log, _ = _run_workers(tmp_path, 2, base + gen, "w2gen")
    r2n, w2n, s2n, _, _ = _run_workers(tmp_path, 2, base, "w2")
    r1, _, _, _, d1 = _run_workers(tmp_path, 1, base + gen, "w1gen")
    assert s2 == s2n and np.array_equal(w2, w2n)
    assert "generations" not in r2n
    assert [g["step"] for g in r2["generations"]] == [2, 4, 5]
    for a, b in zip(r2["generations"], r1["generations"]):
        assert a["tokens"] == b["tokens"] and a["seed"] == b["seed"] and a["text"] == b["text"]
    g = r2["generations"][-1]
    assert len(g["tokens"]) == 3 and all(len(t) == 7 and t[0] == 999 for t in g["tokens"])
    assert g["text"][0] == "".join(_token_bytes(t).decode() for t in g["tokens"][0])
    assert len({g["seed"] for g in r2["generations"]}) == 3
    assert "generation 0:" in log
    assert r2["gpu_launches"] == r2n["gpu_launches"] and r2["launches_per_step"] == r2n["launches_per_step"]
    assert r2["ms_per_step"] < r2n["ms_per_step"] + 500, (r2["ms_per_step"], r2n["ms_per_step"])
    # the checkpoint the one-rank run wrote after its last step, through the command line
    from trainingjob_operator_b200.cmd import generate as cmd

    install_decode(monkeypatch)
    g1 = r1["generations"][-1]
    buf = io.StringIO()
    assert cmd.main(["--cpu", "--model", "gpt2-tiny", "--ckpt", str(d1 / "ckpt" / "gen.pt"), "--prompt", "999",
                     "--tokens", "6", "--count", "3", "--top-k", "40", "--temperature", "0.9", "--seed", str(g1["seed"]),
                     "--tokenizer", tk], out=buf) == 0
    lines = [json.loads(x) for x in buf.getvalue().splitlines()]
    assert [x["tokens"] for x in lines] == g1["tokens"] and [x["text"] for x in lines] == g1["text"]


# ------------------------------------------------------------------------------------ 5. refusals
def _refused(monkeypatch, argv, what):
    from trainingjob_operator_b200.runtime.worker import parse_args

    err = io.StringIO()
    monkeypatch.setattr(sys, "stderr", err)
    with pytest.raises(SystemExit):
        parse_args(argv)
    monkeypatch.undo()
    assert what in err.getvalue(), err.getvalue()


@pytest.mark.parametrize("argv,what", [
    (["--generate-count", "2"], "--generate-count need --generate-every"),
    (["--generate-tokens", "2"], "--generate-tokens need --generate-every"),
    (["--generate-prompt", "1,2"], "--generate-prompt need --generate-every"),
    (["--temperature", "0.5"], "--temperature need --generate-every"),
    (["--top-k", "5"], "--top-k need --generate-every"),
    (["--tokenizer", "t.bin"], "--tokenizer need --generate-every"),
    (["--model", "bert-tiny", "--generate-every", "2"], "GPT-2 models only"),
    (["--generate-every", "-1", "--eot-token", "1"], "cannot be negative"),
    (["--generate-every", "2", "--generate-tokens", "-1", "--eot-token", "1"], "cannot be negative"),
    (["--generate-every", "2", "--temperature", "-0.5", "--eot-token", "1"], "cannot be negative"),
    (["--generate-every", "2", "--top-k", "-3", "--eot-token", "1"], "cannot be negative"),
    (["--generate-every", "2", "--generate-count", "0", "--eot-token", "1"], "at least one sequence"),
    (["--generate-every", "2", "--top-k", "1001", "--eot-token", "1"], "--top-k 1001 exceeds the vocabulary"),
    (["--generate-every", "2", "--generate-tokens", "128", "--eot-token", "1"], "exceed the block size"),
    (["--generate-every", "2", "--generate-prompt", "1,x"], "not a comma-separated list"),
    (["--generate-every", "2", "--generate-prompt", "1,1000"], "--generate-prompt id 1000 is outside the vocabulary"),
    (["--generate-every", "2"], "--eot-token 50256, 50256 is outside the vocabulary"),
])
def test_generation_flags_are_refused_where_they_cannot_run(monkeypatch, argv, what):
    model = [] if "--model" in argv else ["--model", "gpt2-tiny"]
    _refused(monkeypatch, model + argv, what)


def test_generation_flags_take_their_defaults():
    from trainingjob_operator_b200.runtime.worker import parse_args

    a = parse_args(["--model", "gpt2", "--generate-every", "100"])
    assert (a.generate_count, a.generate_tokens, a.generate_prompt, a.temperature, a.top_k) == (4, 64, [50256], 1.0, 0)
    a = parse_args(["--model", "gpt2-tiny"])
    assert a.generate_every is None and a.temperature is None


def test_the_generator_refuses_what_cannot_fit(monkeypatch):
    from trainingjob_operator_b200.models.generate import GPT2Generator

    eng = _engine(monkeypatch)
    with pytest.raises(ValueError, match="max_len 129"):
        GPT2Generator(eng, 2, 129)
    gen = GPT2Generator(eng, 2, 10)
    with pytest.raises(ValueError, match="prompt token id 1000 is outside"):
        gen.generate([3, 1000], 2)
    with pytest.raises(ValueError, match="exceed this generator's max_len 10"):
        gen.generate([3, 4], 9)
    with pytest.raises(ValueError, match="top_k"):
        gen.generate([3], 2, top_k=1001)
    with pytest.raises(ValueError, match="temperature"):
        gen.generate([3], 2, temperature=-1.0)


def _decode_args():
    S, H, T, C = 2, 2, 70, 128
    return dict(
        attention_decode=dict(qkv=torch.zeros(S, 3 * C).bfloat16(), cache=torch.zeros(S, T, 2, H, 64).bfloat16(),
                              pos=torch.zeros(2, dtype=torch.int32), out=torch.zeros(S, C).bfloat16(),
                              part=torch.zeros(F.decode_partials(S, H, T)), H=H),
        embedding_decode=dict(tok=torch.zeros(S, dtype=torch.int64), wte=torch.zeros(50, C).bfloat16(),
                              wpe=torch.zeros(T, C).bfloat16(), pos=torch.zeros(2, dtype=torch.int32),
                              out=torch.zeros(S, C).bfloat16()),
        sample_tokens=dict(logits=torch.zeros(S, 128).bfloat16(), vocab=100, tok=torch.zeros(S, dtype=torch.int64),
                           out_tokens=torch.zeros(S, 8, dtype=torch.int64), prompt=torch.zeros(S, 3, dtype=torch.int64),
                           prompt_len=2, pos=torch.zeros(2, dtype=torch.int32), temperature=1.0, top_k=0, seed=1))


# (entry point, argument, bad value, what the ValueError says)
BAD_DECODE_CALLS = [
    ("attention_decode", "qkv", lambda a: a["qkv"].float(), "qkv must be torch.bfloat16"),
    ("attention_decode", "qkv", lambda a: torch.zeros(0, 384).bfloat16(), "S >= 1"),
    ("attention_decode", "H", lambda a: 3, "H * 64 == C"),
    ("attention_decode", "qkv", lambda a: torch.zeros(2, 3 * 128 + 1).bfloat16()[:, 1:], "contiguous"),
    ("attention_decode", "qkv", lambda a: torch.zeros(2 * 384 + 1).bfloat16()[1:].view(2, 384), "16-byte aligned"),
    ("attention_decode", "cache", lambda a: torch.zeros(2, 70, 2, 2, 32).bfloat16(), "cache must be [S=2"),
    ("attention_decode", "cache", lambda a: torch.zeros(3, 70, 2, 2, 64).bfloat16(), "cache must be [S=2"),
    ("attention_decode", "out", lambda a: torch.zeros(2, 64).bfloat16(), "out must be [2, 128]"),
    ("attention_decode", "part", lambda a: torch.zeros(10), "part must hold"),
    ("attention_decode", "pos", lambda a: torch.zeros(2, dtype=torch.int64), "pos must be torch.int32"),
    ("embedding_decode", "tok", lambda a: torch.zeros(2, dtype=torch.int32), "tok must be torch.int64"),
    ("embedding_decode", "tok", lambda a: torch.zeros(0, dtype=torch.int64), "S >= 1"),
    ("embedding_decode", "wpe", lambda a: torch.zeros(70, 64).bfloat16(), "the same width"),
    ("embedding_decode", "out", lambda a: torch.zeros(3, 128).bfloat16(), "out must be [2, 128]"),
    ("embedding_decode", "pos", lambda a: torch.zeros(0, dtype=torch.int32), "pos must hold at least 1"),
    ("sample_tokens", "logits", lambda a: torch.zeros(2, 128), "2-D bf16"),
    ("sample_tokens", "logits", lambda a: torch.zeros(0, 128).bfloat16(), "S >= 1"),
    ("sample_tokens", "vocab", lambda a: 129, "vocab 129 must be in [1, 128]"),
    ("sample_tokens", "vocab", lambda a: 0, "vocab 0 must be in"),
    ("sample_tokens", "tok", lambda a: torch.zeros(3, dtype=torch.int64), "tok must hold 2"),
    ("sample_tokens", "out_tokens", lambda a: torch.zeros(3, 8, dtype=torch.int64), "out_tokens must have 2 rows"),
    ("sample_tokens", "prompt", lambda a: torch.zeros(2, 3, dtype=torch.int32), "prompt must be torch.int64"),
    ("sample_tokens", "prompt_len", lambda a: 4, "prompt_len 4 must be in [1, 3]"),
    ("sample_tokens", "pos", lambda a: torch.zeros(1, dtype=torch.int32), "pos must hold at least 2"),
    ("sample_tokens", "temperature", lambda a: -0.1, "temperature must be finite and >= 0"),
    ("sample_tokens", "temperature", lambda a: float("inf"), "temperature must be finite and >= 0"),
    ("sample_tokens", "top_k", lambda a: 101, "top_k must be in [0, vocab=100]"),
    ("sample_tokens", "top_k", lambda a: -1, "top_k must be in"),
    ("sample_tokens", "seed", lambda a: -1, "seed must be in"),
]


@pytest.mark.parametrize("fn,arg,bad,what", BAD_DECODE_CALLS, ids=[f"{c[0]}-{c[3][:24]}" for c in BAD_DECODE_CALLS])
def test_the_decode_stand_ins_refuse_what_the_wrappers_refuse(fn, arg, bad, what):
    """Each bad call raises the same ValueError from the wrapper -- before the library is reached, so it runs on any
    machine -- and from the stand-in; the good call is accepted by the stand-in."""
    import re

    args = _decode_args()[fn]
    stand_in = {"attention_decode": attention_decode, "embedding_decode": embedding_decode,
                "sample_tokens": sample_tokens}[fn]
    stand_in(**_decode_args()[fn])
    args[arg] = bad(args)
    messages = []
    for entry in (getattr(F, fn), stand_in):
        with pytest.raises(ValueError, match=re.escape(what)) as e:
            entry(**args)
        messages.append(str(e.value))
    assert messages[0] == messages[1]


# ------------------------------------------------------------------------------------ 6. tokenizer
def test_the_tokenizer_decodes_llmc_files_and_refuses_broken_ones(tmp_path):
    from trainingjob_operator_b200.runtime.tokenizer import Tokenizer, TokenizerError

    t = Tokenizer(_tokenizer_file(tmp_path / "v2.bin", 10))
    assert t.version == 2 and t.eot == 9 and t.vocab_size == 10
    assert t.decode_bytes([1, 7, 0]) == b"<1>\xc3\xa9<0>" and t.decode([1, 7]) == "<1>é"
    assert Tokenizer(_tokenizer_file(tmp_path / "v1.bin", 10, version=1)).eot is None
    with pytest.raises(ValueError, match="token id 10"):
        t.decode([10])
    for name, kw, what in (("magic.bin", dict(magic=20240520), "bad magic 20240520"),
                           ("ver.bin", dict(version=3), "unknown tokenizer version 3"),
                           ("trunc.bin", dict(truncate=2), "truncated at token 9 of 10")):
        path = _tokenizer_file(tmp_path / name, 10, **kw)
        with pytest.raises(TokenizerError, match=f"{name}: {what}"):
            Tokenizer(path)
    (tmp_path / "short.bin").write_bytes(b"\0" * 100)
    with pytest.raises(TokenizerError, match="short.bin: truncated header"):
        Tokenizer(str(tmp_path / "short.bin"))


def test_a_worker_refuses_a_tokenizer_smaller_than_the_vocabulary(monkeypatch, tmp_path):
    from trainingjob_operator_b200.runtime.tokenizer import TokenizerError
    from trainingjob_operator_b200.runtime.worker import EngineAdapter, parse_args

    install_decode(monkeypatch)
    tk = _tokenizer_file(tmp_path / "small.bin", 500)
    args = parse_args(["--model", "gpt2-tiny", "--seq", "128", "--generate-every", "2", "--eot-token", "1",
                       "--tokenizer", tk])
    with pytest.raises(TokenizerError, match="small.bin: 500 tokens, fewer than the 1000"):
        EngineAdapter("gpt2-tiny", 2, 128, args, device="cpu")


# ------------------------------------------------------------------------------------ GPU
def _run_case(name: str, timeout: int = 1200):
    r = subprocess.run([sys.executable, os.path.join(TESTS, "test_generation.py"), name], cwd=ROOT,
                       env=dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, TESTS])), capture_output=True, text=True,
                       timeout=timeout)
    sys.stdout.write(r.stdout[-4000:])
    sys.stderr.write(r.stderr[-2000:])
    assert r.returncode == 0, f"{name} failed:\n{r.stdout[-3000:]}\n{r.stderr[-1500:]}"


def _attention_reference(qkv, cache, p, H):
    """fp64 attention of the new q over cache[:, :p] followed by the new k / v: [S, H * 64]."""
    S, C = qkv.shape[0], H * 64
    q = qkv[:, :C].double().view(S, H, 64)
    k = torch.cat([cache[:, :p, 0].double(), qkv[:, None, C:2 * C].double().view(S, 1, H, 64)], 1)
    v = torch.cat([cache[:, :p, 1].double(), qkv[:, None, 2 * C:].double().view(S, 1, H, 64)], 1)
    w = torch.softmax(torch.einsum("shd,sthd->sht", q, k) / 8.0, -1)
    return torch.einsum("sht,sthd->shd", w, v).reshape(S, C)


def gpu_attention_decode():
    from trainingjob_operator_b200.ops.selfcheck import _check

    Tmax = 1024
    for S in (1, 4, 16):
        for H in (4, 12, 16):
            C = H * 64
            g = torch.Generator(device="cuda").manual_seed(S * 100 + H)
            cache = torch.randn(S, Tmax, 2, H, 64, device="cuda", generator=g).bfloat16()
            part = torch.empty(F.decode_partials(S, H, Tmax), device="cuda")
            for p in (0, 1, 127, 128, 129, 1023):
                qkv = (torch.randn(S, 3 * C, device="cuda", generator=g) * 2).bfloat16()
                pos = torch.tensor([p, 0], dtype=torch.int32, device="cuda")
                before = cache.clone()
                out = torch.empty(S, C, device="cuda").bfloat16()
                F.attention_decode(qkv, cache, pos, out, part, H)
                torch.cuda.synchronize()
                assert torch.equal(cache[:, p, 0].reshape(S, C), qkv[:, C:2 * C]), (S, H, p)
                assert torch.equal(cache[:, p, 1].reshape(S, C), qkv[:, 2 * C:]), (S, H, p)
                keep = torch.ones(Tmax, dtype=torch.bool, device="cuda")
                keep[p] = False
                assert torch.equal(cache[:, keep], before[:, keep]), "attention_decode wrote outside position pos"
                ref = _attention_reference(qkv, before, p, H)
                assert _check(f"attention_decode S={S} H={H} pos={p}", out, ref.float(), 2e-2, atol_scale=5e-2)
                assert int(pos[0]) == p, "attention_decode must not move pos"
    # achieved bandwidth is measured by tools/generate_bench.py
    print("attention_decode ok")


def gpu_sample_tokens():
    from scipy import stats

    V, Vp = 50257, 50304
    g = torch.Generator(device="cuda").manual_seed(0)
    S = 256
    logits = (torch.randn(S, Vp, device="cuda", generator=g) * 3).bfloat16()
    logits[:, V:] = 60.0                                  # padding: larger than any vocabulary logit
    logits[3, 10] = logits[3, 20] = 40.0                  # a tie for the maximum: the lower index wins
    prompt = torch.zeros(S, 1, dtype=torch.int64, device="cuda")
    tok, out = torch.empty(S, dtype=torch.int64, device="cuda"), torch.zeros(S, 2, dtype=torch.int64, device="cuda")
    am = torch.argmax(logits[:, :V].float(), -1)
    for T, k in ((0.0, 0), (1.0, 1), (0.0, 50)):
        pos = torch.zeros(2, dtype=torch.int32, device="cuda")
        F.sample_tokens(logits, V, tok, out, prompt, 1, pos, T, k, 5)
        torch.cuda.synchronize()
        assert torch.equal(tok, am) and torch.equal(out[:, 1], am) and pos.tolist() == [1, 0], (T, k)
    assert int(tok[3]) == 10
    # draws keyed by distinct (sequence, position): 2^17 draws of one row, over top-k, against the restricted softmax
    row = (torch.randn(Vp, device="cuda", generator=g) * 1.5).bfloat16()
    row[V:] = 60.0
    for T, k, n_seq in ((0.8, 40, 128), (1.3, 0, 128)):
        S = n_seq
        lg = row.expand(S, Vp).contiguous()
        tok = torch.empty(S, dtype=torch.int64, device="cuda")
        out = torch.zeros(S, 1, dtype=torch.int64, device="cuda")
        pos = torch.zeros(2, dtype=torch.int32, device="cuda")
        draws = []
        for _ in range(1024):                           # 1024 positions x 128 sequences = 2^17 draws
            F.sample_tokens(lg, V, tok, out, torch.zeros(S, 1, dtype=torch.int64, device="cuda"), 1, pos, T, k, 99)
            draws.append(tok.clone())
        d = torch.cat(draws).cpu()
        assert int(pos[0]) == 1024
        z = row[:V].double().cpu()
        keep = z >= torch.topk(z, k).values[-1] if k else torch.ones(V, dtype=torch.bool)
        assert bool(keep[d].all()) and int(d.max()) < V, "a token outside the top-k or the vocabulary was drawn"
        p = torch.softmax(torch.where(keep, z / T, torch.full_like(z, -float("inf"))), 0)
        counts = torch.bincount(d, minlength=V).double()
        expected = p * d.numel()
        # bins with fewer than 5 expected draws are pooled into one
        big = expected >= 5
        obs = torch.cat([counts[big], counts[~big].sum().view(1)])
        exp = torch.cat([expected[big], expected[~big].sum().view(1)])
        if float(exp[-1]) < 5:
            obs, exp = obs[:-1], exp[:-1] * (obs[:-1].sum() / exp[:-1].sum())
        chi2, pval = stats.chisquare(obs.numpy(), exp.numpy())
        print(f"sample_tokens T={T} top_k={k}: chi2 {chi2:.1f} over {len(obs) - 1} dof, p = {pval:.3g}")
        assert pval > 1e-3, (T, k, chi2, pval)
    print("sample_tokens ok")


def gpu_gpt2_small():
    from trainingjob_operator_b200.models.generate import GPT2Generator
    from trainingjob_operator_b200.models.gpt2 import GPT2Config, GPT2Engine, GPT2Reference

    torch.cuda.set_device(0)
    cfg = GPT2Config.small()
    T = 1024
    eng = GPT2Engine(cfg, 2, T, "cuda", seed=0)
    g = torch.Generator().manual_seed(0)
    tok = torch.randint(0, cfg.vocab_size, (2, T), generator=g)
    eng.tok.copy_(tok.reshape(-1))
    eng._trunk()
    eng._linear(eng.lnf, eng.params.w16("wte"), eng.logits)
    fwd = eng.logits[:, :cfg.vocab_size].float().view(2, T, -1)[:, :T - 1].clone()
    ref = GPT2Reference(cfg, eng.params).cuda()
    import torch.nn.functional as TF

    seen = {}
    ce = TF.cross_entropy
    TF.cross_entropy = lambda z, t: seen.setdefault("z", z).sum()
    with torch.no_grad():
        ref(tok.cuda(), tok.cuda())
    TF.cross_entropy = ce
    want = seen["z"].view(2, T, -1)[:, :T - 1]
    gen = GPT2Generator(eng, 2, T)
    got = torch.empty(2, T - 1, cfg.vocab_size, device="cuda")
    out = gen.generate(tok, 0, temperature=0.0, logits_out=got)
    assert torch.equal(out, tok)
    e_dec, e_fwd = float((got - want).abs().max()), float((fwd - want).abs().max())
    print(f"GPT-2 small teacher-forced over {T} positions: max |decode - fp32| {e_dec:.4f}, "
          f"max |forward - fp32| {e_fwd:.4f}")
    assert e_dec <= 1.5 * e_fwd, (e_dec, e_fwd)
    del got, fwd, want, ref, seen
    prompt = [50256, 464, 3290]
    g8 = GPT2Generator(eng, 8, 200)
    graph = g8.generate(prompt, 190, temperature=1.0, top_k=50, seed=3)
    eager = g8.generate(prompt, 190, temperature=1.0, top_k=50, seed=3, use_graph=False)
    assert torch.equal(graph, eager), "graph replay and eager decoding differ"
    g1 = GPT2Generator(eng, 1, 200)
    for i in (0, 5):
        assert torch.equal(g1.generate(prompt, 190, temperature=1.0, top_k=50, seed=3, first_seq=i)[0], graph[i])
    greedy8 = g8.generate(prompt, 50, temperature=0.0)
    assert torch.equal(g1.generate(prompt, 50, temperature=0.0, first_seq=7)[0], greedy8[7])
    print("GPT-2 small generation ok")


@pytest.mark.gpu
def test_attention_decode_against_fp64():
    _run_case("gpu_attention_decode")


@pytest.mark.gpu
def test_sample_tokens_greedy_top_k_and_distribution():
    _run_case("gpu_sample_tokens")


@pytest.mark.gpu
def test_gpt2_small_decodes_like_the_training_forward():
    _run_case("gpu_gpt2_small")


def _gpu_worker(argv, timeout=900):
    env = dict(os.environ, WORLD_SIZE="1", RANK="0", PYTHONPATH=ROOT)
    env.pop("AITJ_MASTER", None)
    r = subprocess.run([sys.executable, "-m", "trainingjob_operator_b200.runtime.worker"] + argv, cwd=ROOT, env=env,
                       capture_output=True, text=True, timeout=timeout)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    return r.stdout


@pytest.mark.gpu
def test_one_gpu_worker_generates_without_changing_its_training(tmp_path):
    """On the GPU the training step itself is not bitwise reproducible from run to run -- split-K weight-gradient
    GEMMs, LayerNorm-backward and embedding-backward add into the gradients with atomics; two runs of 22 steps at
    lr 1e-3 were measured 3e-4 apart in loss and 1.1e-2 in a weight -- so the run with generation is held to that
    spread; the CPU worker test holds it to bit equality."""
    train = write_llmc(tmp_path / "train_000.bin", structured_corpus(400000, 1000, 999, 0))
    base = ["--model", "gpt2-tiny", "--batch", "8", "--seq", "128", "--steps", "20", "--warmup", "2", "--lr", "1e-3",
            "--data", train, "--eot-token", "999"]
    runs = {}
    for tag, extra in (("gen", ["--generate-every", "10", "--generate-tokens", "32", "--top-k", "20"]), ("plain", [])):
        out = tmp_path / tag
        log = _gpu_worker(base + extra + ["--result", str(out / "r.json"), "--dump-outputs", str(out / "dump")])
        runs[tag] = (json.load(open(out / "r.json")), np.load(out / "dump" / "losses.npy"),
                     np.load(out / "dump" / "weights_sample.npy"), log)
    (rg, lg, wg, log), (rp, lp, wp, _) = runs["gen"], runs["plain"]
    print(json.dumps({k: rg[k] for k in ("ms_per_step", "generations")})[:3000])
    assert [x["step"] for x in rg["generations"]] == [10, 20, 22]
    assert all(len(t) == 33 for x in rg["generations"] for t in x["tokens"])
    assert np.allclose(lg, lp, rtol=2e-3, atol=0) and np.allclose(wg, wp, rtol=0, atol=3e-2), \
        ("generation changed the training", float(np.abs(lg - lp).max()), float(np.abs(wg - wp).max()))
    assert rg["cuda_graph"] and "generation 0:" in log and "generations" not in rp


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
                   "--lr", "1e-3", "--eot-token", "999", "--generate-every", "2", "--generate-tokens", "40"])
a = EngineAdapter("gpt2-tiny", 4, 128, args)
a.bind(None)
recs = [a.generate(0)]
for _ in range(3):
    a.train_step()
recs.append(a.generate(3))
json.dump(recs, open(os.path.join({out!r}, f"w{{world}}_{{rank}}.json"), "w"))
if world > 1:
    dist.destroy_process_group()
"""


@pytest.mark.gpu
@pytest.mark.gpu2
def test_two_gpus_generate_what_one_does(tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    train = write_llmc(tmp_path / "train_000.bin", structured_corpus(200000, 1000, 999, 2))
    script = tmp_path / "gen2.py"
    script.write_text(TWO_GPU_SCRIPT.format(root=ROOT, train=train, out=str(tmp_path)))
    port = _free_port()
    for world in (1, 2):
        procs = [subprocess.Popen([sys.executable, str(script)], cwd=ROOT, stdout=subprocess.PIPE,
                                  stderr=subprocess.STDOUT, text=True,
                                  env=dict(os.environ, RANK=str(r), WORLD_SIZE=str(world), MASTER_ADDR="127.0.0.1",
                                           MASTER_PORT=str(port + world)))
                 for r in range(world)]
        logs = [p.communicate(timeout=900)[0] for p in procs]
        assert all(p.returncode == 0 for p in procs), "\n".join(l[-3000:] for l in logs)
    # the ranks hold the same weights, so they generate the same; one GPU generates the same at step 0 (after
    # training, the two worlds' weights differ by the order of their gradient sums)
    one = json.load(open(tmp_path / "w1_0.json"))
    two = [json.load(open(tmp_path / f"w2_{r}.json")) for r in range(2)]
    assert two[0] == two[1]
    assert two[0][0]["tokens"] == one[0]["tokens"] and two[0][0]["seed"] == one[0]["seed"]


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    globals()[sys.argv[1]]()
