"""The decode kernels (``ops/csrc/decode.cu``) and the GEMMs of a decode step against references of the same operation,
at every GPT-2 size and at the shapes where they can go wrong.

* ``sample_tokens`` draw by draw: every draw recomputes its Philox word in numpy, and the fp64 distribution over the
  kept columns says which tokens that word may give (``draw_intervals``, ``sampling_delta``).  A float32 model of the
  kernel's scan (``scan_model``) reproduces, on the CPU, rows whose draws an earlier kernel left unclaimed.
* ``attention_decode`` against fp64 at H 12 / 16 / 20 / 25, cache lengths that are and are not multiples of the 64-key
  chunk, and positions on both sides of a chunk boundary, with the partials' scratch filled with NaN first.
* ``embedding_decode`` bit for bit.
* The five GEMMs of a decode step at M = 1 .. 65 rows, each output a view of the first M rows of a larger buffer whose
  other rows must keep a sentinel.

CPU tests check the oracles themselves; the GPU cases run one per process (``_run_case``)."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from test_generation import _attention_reference, philox_first_word
from test_generation import sample_tokens as sample_tokens_stand_in

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTS = os.path.dirname(os.path.abspath(__file__))

SAMPLE_THREADS = 1024                                  # kSampleThreads of decode.cu: one run of columns per thread
LOG2E_F32 = float(np.float32(1.4426950408889634))     # at this temperature the kernel's exp2 scale is exactly 1.0f
M32 = np.uint64(0xFFFFFFFF)


# ------------------------------------------------------------------------------------ Philox, vectorised
def philox_first_words(seed: int, seq, pos) -> np.ndarray:
    """``philox_first_word`` over numpy arrays of sequences and positions (broadcast): uint64 words < 2^32."""
    c0, c1 = np.broadcast_arrays(np.asarray(pos, np.uint64) & M32, np.asarray(seq, np.uint64) & M32)
    c0, c1 = c0.copy(), c1.copy()
    c2, c3 = np.zeros_like(c0), np.zeros_like(c0)
    k0, k1 = np.uint64(seed & 0xFFFFFFFF), np.uint64((seed >> 32) & 0xFFFFFFFF)
    for _ in range(10):
        p0, p1 = np.uint64(0xD2511F53) * c0, np.uint64(0xCD9E8D57) * c2
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & M32, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & M32
        k0, k1 = (k0 + np.uint64(0x9E3779B9)) & M32, (k1 + np.uint64(0xBB67AE85)) & M32
    return c0


def draw_u(seed: int, seq, pos) -> np.ndarray:
    """The uniform of each draw, as the kernel forms it: (word >> 8) / 2^24."""
    return (philox_first_words(seed, seq, pos) >> np.uint64(8)).astype(np.float64) / float(1 << 24)


# ------------------------------------------------------------------------------------ the per-draw oracle
def draw_intervals(z, temperature: float, top_k: int):
    """fp64 (w, lo, hi) [R, V] of the logits z [R, V] (the bf16 values, exactly): the unnormalised probability of every
    column, and the CDF interval [lo, hi) a draw's u must fall in to give that column.  Greedy (temperature 0 or top_k
    1) puts all the mass on the first maximum; otherwise columns below the top_k-th largest (ties kept) have none."""
    z = z.double()
    if temperature == 0 or top_k == 1:
        w = torch.zeros_like(z).scatter_(1, torch.argmax(z, 1, keepdim=True), 1.0)
    else:
        V = z.shape[1]
        keep = z >= torch.topk(z, top_k, 1).values[:, -1:] if 0 < top_k < V else torch.ones_like(z, dtype=torch.bool)
        t = float(np.float32(temperature))                    # the kernel receives an fp32 temperature
        w = torch.where(keep, torch.exp((z - z.max(1, keepdim=True).values) / t), torch.zeros_like(z))
    c = torch.cumsum(w, 1)
    tot = c[:, -1:]
    return w, (c - w) / tot, c / tot


def sampling_delta(z, w, temperature: float) -> torch.Tensor:
    """Per row, how far the kernel's choice may sit from the fp64 CDF interval of its token, in u.

    The kernel draws target = fl(u * total) and walks fp32 prefix sums of fp32 terms e_c = exp2f(fl(fl(z_c - zmax) *
    scale)), scale = fl(fl(log2 e) / T).  Three things move its boundaries from the fp64 CDF's:

    * summation.  Any prefix it compares is a sum of nonnegative terms formed by at most 50 serial adds in a thread's
      run (ceil(50257 / 1024) columns), 5 warp-scan levels, one add of the warps below and 5 levels of their scan, then
      up to 50 adds of the owner's walk, plus the rounding of u * total: n = 112 roundings on any path.  The standard
      bound for such sums is n * 2^-24 of the total, 6.7e-6.
    * exp2f: at most 2 ulp (CUDA C Programming Guide, maximum ulp error of exp2f), 2.4e-7 of every term, so of every
      prefix and of the total.
    * the argument: fl(z - zmax), the two roundings of the scale and that of the product are 4 * 2^-24 of |a| for
      a = (z - zmax) log2(e) / T, which moves the term by ln 2 |a| 4 * 2^-24 of itself: over the row, ln 2 * 4 * 2^-24
      times the mean of |a| weighted by the terms.  This one depends on the row and is computed from it.

    A boundary is a prefix over the total, both off by at most eps of the total, so it moves by 2 eps:
    delta = 2 (112 * 2^-24 + 2.4e-7 + argument term): 1.4e-5 plus the argument term, a few 1e-6 for these rows."""
    ulp = 2.0 ** -24
    if temperature == 0:
        return torch.full((z.shape[0],), 2 * (112 * ulp + 2.4e-7), dtype=torch.float64, device=z.device)
    a = (z.double() - z.double().max(1, keepdim=True).values).abs() * (1.4426950408889634 / float(np.float32(temperature)))
    wa = torch.where(w > 0, w * a, torch.zeros_like(w)).sum(1) / w.sum(1)
    return 2 * (112 * ulp + 2.4e-7 + math.log(2) * 4 * ulp * wa)


def wrong_draws(tok, u, w, lo, hi, delta, vocab: int) -> torch.Tensor:
    """bool [R, P]: draws tok [R, P] with uniforms u [R, P] that the oracle does not allow -- a column outside the
    vocabulary, one with no probability (not kept, or -inf), or one whose interval is more than delta from u."""
    tok, u = tok.to(w.device), u.to(w.device)
    inside = (tok >= 0) & (tok < vocab)
    t = tok.clamp(0, vocab - 1)
    d = delta.view(-1, 1)
    ok = inside & (w.gather(1, t) > 0) & (u >= lo.gather(1, t) - d) & (u <= hi.gather(1, t) + d)
    return ~ok


# ------------------------------------------------------------------------------------ float32 model of the scan
def bf16_bits(z) -> np.ndarray:
    return (np.asarray(z, np.float32).view(np.uint32) >> 16).astype(np.uint16)


def thread_scan(part: np.ndarray):
    """The kernel's float32 inclusive scan over 1024 thread parts (Hillis-Steele in each warp, then over the warp
    sums, added to the warps above): (incl, excl = incl - part, total = the last warp sum's scan)."""
    incl = part.astype(np.float32).reshape(-1, 32).copy()
    for o in (1, 2, 4, 8, 16):
        nxt = incl.copy()
        nxt[:, o:] = incl[:, o:] + incl[:, :-o]
        incl = nxt
    w = incl[:, 31].copy()
    for o in (1, 2, 4, 8, 16):
        nxt = w.copy()
        nxt[o:] = w[o:] + w[:-o]
        w = nxt
    incl[1:] += w[:-1, None]
    incl = incl.reshape(-1)
    return incl, (incl - part).astype(np.float32), np.float32(w[-1])


def scan_model(bits: np.ndarray, temperature: float):
    """float32 model of ``sample_tokens_kernel`` at top_k = 0 over one bf16 row: each thread's part (its run summed in
    order) and ``thread_scan``.  exp2 of an integer is taken to be exact in exp2f too, as it is in numpy."""
    z = (bits.astype(np.uint32) << 16).view(np.float32)
    scale = np.float32(1.4426950408889634) / np.float32(temperature)
    terms = np.exp2((z - z.max()) * scale).astype(np.float32)
    per = -(-bits.size // SAMPLE_THREADS)
    part = np.zeros(SAMPLE_THREADS, np.float32)
    for t in range(SAMPLE_THREADS):
        for c in range(min(bits.size, t * per), min(bits.size, t * per + per)):
            part[t] = np.float32(part[t] + terms[c])
    incl, excl, total = thread_scan(part)
    return dict(terms=terms, part=part, incl=incl, excl=excl, total=total, per=per)


def model_target(m, u24: int) -> np.float32:
    t = np.float32(np.float32(u24) * np.float32(1.0 / 16777216.0)) * m["total"]
    return t if t < m["total"] else np.nextafter(m["total"], np.float32(0))


def model_claimants(m, target) -> list:
    """Threads the earlier kernel let claim the target: a kept column and excl <= target < incl."""
    return [int(t) for t in np.nonzero((m["part"] > 0) & (m["excl"] <= target) & (target < m["incl"]))[0]]


def model_owner_token(m, target) -> int:
    """The token the kernel draws: the owner is the last thread with a kept column and excl <= target; it walks its
    run from excl and takes the first column whose running sum passes the target (else its last nonzero one)."""
    owner = int(np.nonzero((m["part"] > 0) & (m["excl"] <= target))[0].max())
    acc, last = m["excl"][owner], -1
    for c in range(owner * m["per"], min(len(m["terms"]), owner * m["per"] + m["per"])):
        if m["terms"][c] > 0:
            last = c
        acc = np.float32(acc + m["terms"][c])
        if target < acc:
            return c
    return last


def gap_row() -> np.ndarray:
    """bf16 bits of 1024 integer logits (one column per thread): 0 at column 0, -1 .. -31 elsewhere, -inf at every
    37th column from 5.  At temperature LOG2E_F32 every term is a power of two, so the float32 model is exact."""
    c = np.arange(1024)
    z = -((c * c * 7 + c * 3) % 31).astype(np.float32) - 1
    z[c % 37 == 5] = -np.inf
    z[0] = 0
    return bf16_bits(z)


# (sequence, position, word >> 8) under GAP_SEED whose target falls between two threads' intervals of the gap row in
# the earlier kernel's scan (found by searching 64 sequences x 65536 positions with ``philox_first_words``)
GAP_SEED = 20261018
GAP_DRAWS = [(8, 54281, 11149615), (12, 22502, 8117837), (20, 40712, 15232896), (27, 40374, 16536903),
             (40, 4892, 16026673)]


def zero_tie_row() -> torch.Tensor:
    """1000 logits whose 40th largest is +0 and 500 of which are -0: with top_k 40 every -0 ties with the threshold
    and is kept, and they hold most of the mass."""
    z = torch.full((1000,), -3.0)
    z[100:139] = torch.linspace(0.5, 1.0, 39)
    z[200:700] = -0.0
    z[700] = 0.0
    return z.bfloat16()


# ------------------------------------------------------------------------------------ CPU tests of the oracles
def test_the_vectorised_philox_equals_the_scalar_one():
    rng = np.random.default_rng(0)
    seeds = [0, 1, 5, 99, 2 ** 32 - 1, 2 ** 32, 2 ** 63 - 1, GAP_SEED] + [int(x) for x in rng.integers(0, 2 ** 63, 4)]
    seq = np.concatenate([[0, 1, 2 ** 31 - 1, 2 ** 32 - 1], rng.integers(0, 2 ** 32, 60)]).astype(np.uint64)
    pos = np.concatenate([[0, 1, 1023, 2 ** 32 - 1], rng.integers(0, 2 ** 32, 60)]).astype(np.uint64)
    for seed in seeds:
        got = philox_first_words(seed, seq[:, None], pos[None, :])
        want = [[philox_first_word(seed, int(s), int(p)) for p in pos] for s in seq]
        assert np.array_equal(got, np.array(want, np.uint64)), seed


def test_the_oracle_takes_a_draw_within_delta_of_its_interval_and_nothing_else():
    z = torch.tensor([[0.0, math.log(2.0), -math.inf, 0.0, -5.0]])
    w, lo, hi = draw_intervals(z, 1.0, 0)                   # masses 1, 2, 0, 1, e^-5
    tot = 4 + math.exp(-5)
    assert torch.allclose(hi[0, :4], torch.tensor([1, 3, 3, 4], dtype=torch.float64) / tot)
    d = torch.tensor([1e-5], dtype=torch.float64)
    edge = float(hi[0, 0])

    def wrong(tok, u, vocab=5):
        return bool(wrong_draws(torch.tensor([[tok]]), torch.tensor([[u]], dtype=torch.float64), w, lo, hi, d, vocab))

    assert not wrong(0, edge + 0.5e-5) and wrong(0, edge + 2e-5)     # just past column 0's interval: within delta
    assert not wrong(1, edge - 0.5e-5) and wrong(1, edge - 2e-5)
    assert not wrong(1, 0.5) and wrong(0, 0.5) and wrong(3, 0.5)
    assert wrong(2, float(lo[0, 2]))                                 # no probability: never, even at its point
    assert wrong(5, 0.5) and wrong(-1, 0.0) and wrong(4, 0.5, vocab=4)
    # top_k keeps ties with the k-th, including -0 against +0; greedy is the first maximum
    z2 = torch.tensor([[1.0, 0.0, -0.0, 0.0, -1.0, 1.0]])
    w2, _, _ = draw_intervals(z2, 0.7, 3)
    assert (w2[0] > 0).tolist() == [True, True, True, True, False, True]
    assert (draw_intervals(z2, 0.7, 1)[0][0] > 0).tolist() == [True] + [False] * 5
    assert (draw_intervals(z2, 0.0, 0)[0][0] > 0).tolist() == [True] + [False] * 5
    # the bound: 1.4e-5 from the sums and exp2f, plus the argument term, which grows with the spread of the terms
    zr = torch.randn(4, 50257, generator=torch.Generator().manual_seed(0)).mul(3).bfloat16().float()
    for T in (1e-3, 0.7, 1.0, 2.5):
        delta = sampling_delta(zr, draw_intervals(zr, T, 0)[0], T)
        assert bool((delta > 1.38e-5).all()) and bool((delta < 2.5e-5).all()), (T, delta)


def test_the_scan_model_leaves_the_gap_rows_targets_to_no_thread():
    """The earlier kernel let thread t claim a target in [incl - part, incl); for these draws of ``gap_row`` no thread
    does, so it returned the argmax (column 0).  The owner rule gives each a column next to the fp64 CDF's."""
    bits = gap_row()
    m = scan_model(bits, LOG2E_F32)
    z = torch.from_numpy((bits.astype(np.uint32) << 16).view(np.float32).copy())[None]
    w, lo, hi = draw_intervals(z, LOG2E_F32, 0)
    delta = sampling_delta(z, w, LOG2E_F32)
    for seq, pos, word in GAP_DRAWS:
        assert int(philox_first_words(GAP_SEED, seq, pos)) >> 8 == word
        target = model_target(m, word)
        assert model_claimants(m, target) == [], (seq, pos)
        u = torch.tensor([[word / float(1 << 24)]], dtype=torch.float64)
        assert bool(wrong_draws(torch.tensor([[0]]), u, w, lo, hi, delta, 1024)), "the argmax would pass the oracle"
        assert not bool(wrong_draws(torch.tensor([[model_owner_token(m, target)]]), u, w, lo, hi, delta, 1024))


def test_predecessor_tiling_alone_would_still_overlap():
    """Why the kernel picks one owner instead of taking each thread's exclusive prefix from its predecessor: the
    tree-ordered scan is not monotone.  Parts 1, 2^-24, 2^-24, 0, 1 give incl_2 = 1 + 2^-23 but incl_3 = 1, so thread 4
    would start at 1 and overlap thread 2's [1, 1 + 2^-23)."""
    part = np.zeros(SAMPLE_THREADS, np.float32)
    part[:5] = [1.0, 2.0 ** -24, 2.0 ** -24, 0.0, 1.0]
    incl, _, _ = thread_scan(part)
    assert incl[2] == np.float32(1 + 2.0 ** -23) and incl[3] == np.float32(1.0) and incl[3] < incl[2]


def test_the_stand_in_keeps_negative_zeros_tied_with_the_threshold():
    z = zero_tie_row()
    S = 64
    logits = z.expand(S, -1).contiguous()
    tok, out = torch.zeros(S, dtype=torch.int64), torch.zeros(S, 2, dtype=torch.int64)
    sample_tokens_stand_in(logits, 1000, tok, out, torch.zeros(S, 1, dtype=torch.int64), 1, torch.zeros(2, dtype=torch.int32),
                           1.0, 40, 7)
    neg = torch.signbit(z.float()) & (z.float() == 0)
    assert int(neg.sum()) == 500 and bool(neg[tok].any()), "no draw took a -0 column"
    w, lo, hi = draw_intervals(logits.float(), 1.0, 40)
    u = torch.from_numpy(draw_u(7, np.arange(S), 0)).view(S, 1)
    assert not bool(wrong_draws(tok.view(S, 1), u, w, lo, hi, sampling_delta(logits.float(), w, 1.0), 1000).any())


# ------------------------------------------------------------------------------------ GPU cases
def _run_case(name: str, timeout: int = 1200):
    r = subprocess.run([sys.executable, os.path.join(TESTS, "test_decode_kernels.py"), name], cwd=ROOT,
                       env=dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, TESTS])), capture_output=True, text=True,
                       timeout=timeout)
    sys.stdout.write(r.stdout[-6000:])
    sys.stderr.write(r.stderr[-2000:])
    assert r.returncode == 0, f"{name} failed:\n{r.stdout[-3000:]}\n{r.stderr[-1500:]}"


def _sample_rows(S: int, V: int, Vp: int, seed: int) -> torch.Tensor:
    """bf16 [S, Vp] logits on the GPU.  Every row has -inf entries and padding columns (>= V) larger than any logit;
    row s % 4 == 1 has a tie of ten equal values straddling the 40th largest, row s % 4 == 2 has 39 positive values
    and then +0 and -0 columns, so that the 40th largest is a zero, and row s % 4 == 3 has a quarter of its columns at
    -inf and its maximum twice, in two different warps' columns."""
    g = torch.Generator().manual_seed(seed)
    z = torch.randn(S, V, generator=g) * 3
    for s in range(S):
        if V >= 100 and s % 4 == 1:
            idx = torch.argsort(z[s], descending=True)
            z[s, idx[35:45]] = float(z[s, idx[39]])
        elif V >= 1000 and s % 4 == 2:
            z[s] = -z[s].abs() - 0.01
            cols = torch.randperm(V, generator=g)
            z[s, cols[:39]] = z[s, cols[:39]].abs() + 0.5
            z[s, cols[39:239]] = 0.0
            z[s, cols[239:439]] = -0.0
        elif V >= 100 and s % 4 == 3:
            z[s, torch.randperm(V, generator=g)[:V // 4]] = -math.inf
            z[s, 37] = z[s, V - 101] = float(z[s].max()) + 1.0     # warp 1, and warp 31 (50257) or 28 (1000)
        if V >= 100:
            z[s, torch.randint(0, V, (5,), generator=g)] = -math.inf
    out = torch.full((S, Vp), 60.0)
    out[:, :V] = z
    return out.bfloat16().cuda()


def _draw(logits, V, T, k, seed, first_seq, P, p0=0):
    """P launches of F.sample_tokens from position p0: the tokens [S, P] (gathered through out_tokens, ld P + 1) and
    the pos after every launch [P, 2]."""
    from trainingjob_operator_b200.ops import functional as F

    S = logits.shape[0]
    tok = torch.empty(S, dtype=torch.int64, device="cuda")
    out = torch.full((S, p0 + P + 1), -7, dtype=torch.int64, device="cuda")
    prompt = torch.zeros(S, 1, dtype=torch.int64, device="cuda")
    pos = torch.tensor([p0, 0], dtype=torch.int32, device="cuda")
    hist = torch.empty(P, 2, dtype=torch.int32, device="cuda")
    for i in range(P):
        F.sample_tokens(logits, V, tok, out, prompt, 1, pos, T, k, seed, first_seq)
        hist[i].copy_(pos)
    torch.cuda.synchronize()
    assert torch.equal(out[:, :p0 + 1], torch.full_like(out[:, :p0 + 1], -7)), "a column before p0 + 1 was written"
    assert torch.equal(out[:, p0 + P], tok)
    want = torch.stack([torch.arange(p0 + 1, p0 + P + 1), torch.zeros(P, dtype=torch.int64)], 1).int().cuda()
    assert torch.equal(hist, want), "pos did not advance by exactly 1 per launch, or pos[1] was not 0 again"
    return out[:, p0 + 1:], hist


def _oracle_count(logits, V, T, k, seed, first_seq, tokens, p0=0):
    """Draws [S, P] (positions p0 ..) the fp64 oracle does not allow."""
    S, P = tokens.shape
    z = logits[:, :V].double()
    w, lo, hi = draw_intervals(z, T, k)
    delta = sampling_delta(z, w, T)
    assert float(delta.max()) < 2.5e-5, float(delta.max())
    u = torch.from_numpy(draw_u(seed, first_seq + np.arange(S)[:, None], p0 + np.arange(P)[None, :])).cuda()
    return wrong_draws(tokens, u, w, lo, hi, delta, V)


def gpu_sample_tokens_oracle():
    """2^20 and more draws, each against the fp64 oracle of its own Philox word, at V 50257 (padded to 50304), 1000
    and 1, every top_k in {0, 1, 40, V} and temperature in {1e-3, 0.7, 1.0, 2.5}, S 1 and 264 (two rows per SM),
    first_seq 0 and not."""
    draws = bad = 0
    for V, Vp, P in ((50257, 50304, 384), (1000, 1024, 64), (1, 8, 8)):
        rows = _sample_rows(264, V, Vp, seed=V)
        ks = (0, 1, 40, V) if V > 40 else (0, 1)
        i = 0
        for T in (1e-3, 0.7, 1.0, 2.5):
            for k in ks:
                logits = rows[i:i + 1] if i % 4 == 3 else rows
                first_seq = 0 if i % 2 == 0 else 1000 + 7 * i
                seed = 7 * V + i
                tokens, _ = _draw(logits, V, T, k, seed, first_seq, P)
                wrong = _oracle_count(logits, V, T, k, seed, first_seq, tokens)
                n = int(wrong.sum())
                where = ""
                if n:
                    s, p = wrong.nonzero()[0].tolist()
                    where = f" first at row {s} position {p}: token {int(tokens[s, p])}"
                print(f"sample_tokens V={V} T={T} top_k={k} S={logits.shape[0]} first_seq={first_seq}: "
                      f"{n} of {tokens.numel()} draws outside the oracle{where}", flush=True)
                draws += tokens.numel()
                bad += n
                i += 1
    print(f"sample_tokens oracle: {bad} wrong of {draws} draws")
    assert draws >= 1 << 20
    assert bad == 0


def gpu_sample_tokens_contracts():
    from trainingjob_operator_b200.ops import functional as F

    # top_k = V draws what top_k = 0 draws
    for V, Vp in ((50257, 50304), (1000, 1024)):
        rows = _sample_rows(264, V, Vp, seed=V + 1)
        a, _ = _draw(rows, V, 0.9, 0, 11, 5, 32)
        b, _ = _draw(rows, V, 0.9, V, 11, 5, 32)
        assert torch.equal(a, b), f"top_k={V} and top_k=0 draw differently"
    # greedy: the first maximum, with the tied pair in different warps (column c is staged by thread c % 1024) or in
    # one thread; at temperature 1e-3 a unique maximum is the only draw, and a tied one splits the draws
    V, Vp = 50257, 50304
    pairs = [(5000, 40000), (40000, 45000), (33, 2), (7, 7 + 1024), (50255, 50256), (0, 50256)]
    logits = _sample_rows(len(pairs) + 2, V, Vp, seed=3)
    for r, (a, b) in enumerate(pairs):
        logits[r, a] = logits[r, b] = 30.0
    logits[len(pairs), 12345] = 30.0                              # a unique maximum
    want = torch.tensor([min(p) for p in pairs] + [12345, int(torch.argmax(logits[-1, :V].float()))], device="cuda")
    for T, k in ((0.0, 0), (1.0, 1), (0.0, 40)):
        got, _ = _draw(logits, V, T, k, 1, 0, 2)
        assert torch.equal(got, want[:, None].expand(-1, 2)), (T, k, got[:, 0].tolist(), want.tolist())
    got, _ = _draw(logits, V, 1e-3, 0, 2, 0, 256)
    assert bool((got[len(pairs)] == 12345).all())
    for r, (a, b) in enumerate(pairs):
        assert set(got[r].tolist()) == {a, b}, (r, sorted(set(got[r].tolist())))
    # prompt forcing: positions p < prompt_len - 1 give prompt[s, p + 1] whatever the logits (NaN here, never read)
    S, L = 264, 8
    prompt = torch.randint(0, V, (S, L), device="cuda")
    prompt[:, 1], prompt[:, 2] = 0, V - 1
    nan = torch.full((S, Vp), float("nan"), device="cuda").bfloat16()
    tok = torch.empty(S, dtype=torch.int64, device="cuda")
    buf = torch.full((S * 3 + 16,), -5, dtype=torch.int64, device="cuda")
    out = buf[:S * 3].view(S, 3)                                  # ld_out 3: positions 0 and 1 only are stored
    pos = torch.zeros(2, dtype=torch.int32, device="cuda")
    forced = []
    for p in range(5):
        F.sample_tokens(nan, V, tok, out, prompt, 6, pos, 1.0, 40, 9)
        forced.append(tok.clone())
    torch.cuda.synchronize()
    for p in range(5):
        assert torch.equal(forced[p], prompt[:, p + 1]), f"position {p} did not return the prompt's token"
    assert torch.equal(out[:, 1], prompt[:, 1]) and torch.equal(out[:, 2], prompt[:, 2])
    assert bool((out[:, 0] == -5).all()) and bool((buf[S * 3:] == -5).all()), "out_tokens written past ld_out"
    # the first position past the prompt samples from the logits
    rows = _sample_rows(S, V, Vp, seed=4)
    F.sample_tokens(rows, V, tok, out, prompt, 6, pos, 0.0, 0, 9)
    torch.cuda.synchronize()
    assert torch.equal(tok, torch.argmax(rows[:, :V].float(), 1)) and pos.tolist() == [6, 0]
    assert bool((out[:, 0] == -5).all()) and bool((buf[S * 3:] == -5).all())
    # pos moves on from a nonzero start with more CTAs than SMs (checked inside _draw)
    _draw(rows, V, 1.0, 0, 3, 0, 16, p0=1000)
    print("sample_tokens contracts ok")


def gpu_sample_tokens_regressions():
    """Two fixed rows whose draws an earlier kernel got wrong: -0 columns tied with a +0 40th largest were dropped, and
    draws of ``gap_row`` at the GAP_DRAWS counters fell between two threads' intervals and returned the argmax."""
    fails = []
    z = zero_tie_row()
    S = 64
    logits = torch.full((S, 1024), 60.0).bfloat16()
    logits[:, :1000] = z
    logits = logits.cuda()
    tokens, _ = _draw(logits, 1000, 1.0, 40, 7, 0, 4)
    wrong = _oracle_count(logits, 1000, 1.0, 40, 7, 0, tokens)
    neg = torch.signbit(z.float()) & (z.float() == 0)
    print(f"-0 tie row: {int(wrong.sum())} of {tokens.numel()} draws outside the oracle, "
          f"{int(neg.cuda()[tokens].sum())} in -0 columns")
    if int(wrong.sum()):
        fails.append("-0 tie row")
    bits = torch.from_numpy(gap_row().view(np.int16)).view(torch.bfloat16)
    row = torch.full((1, 1024 + 8), 60.0).bfloat16()
    row[0, :1024] = bits
    row = row.cuda()
    from trainingjob_operator_b200.ops import functional as F

    tok = torch.empty(1, dtype=torch.int64, device="cuda")
    out = torch.full((1, 1), -7, dtype=torch.int64, device="cuda")
    prompt = torch.zeros(1, 1, dtype=torch.int64, device="cuda")
    z64 = row[:, :1024].double()
    w, lo, hi = draw_intervals(z64, LOG2E_F32, 0)
    delta = sampling_delta(z64, w, LOG2E_F32)
    for seq, p, word in GAP_DRAWS:
        pos = torch.tensor([p, 0], dtype=torch.int32, device="cuda")
        F.sample_tokens(row, 1024, tok, out, prompt, 1, pos, LOG2E_F32, 0, GAP_SEED, seq)
        torch.cuda.synchronize()
        u = torch.tensor([[word / float(1 << 24)]], dtype=torch.float64)
        bad = bool(wrong_draws(tok.view(1, 1), u, w, lo, hi, delta, 1024))
        t = int(tok)
        print(f"gap row seq={seq} pos={p}: token {t}, oracle interval of u {word / 2 ** 24:.8f} in column "
              f"{int(torch.searchsorted(hi[0].cpu(), torch.tensor([word / 2 ** 24], dtype=torch.float64)))}"
              f"{' WRONG' if bad else ''}")
        assert pos.tolist() == [p + 1, 0] and int(out[0, 0]) == -7
        if bad:
            fails.append(f"gap row seq={seq}")
    assert not fails, fails
    print("sample_tokens regressions ok")


def gpu_attention_decode_sizes():
    from trainingjob_operator_b200.ops import functional as F
    from trainingjob_operator_b200.ops.selfcheck import _check

    ok = True
    for H in (12, 16, 20, 25):
        C = H * 64
        for Tmax in (200, 1000, 1024):
            for S in (1, 3, 16):
                g = torch.Generator(device="cuda").manual_seed(H * 10000 + Tmax * 10 + S)
                cache = torch.randn(S, Tmax, 2, H, 64, device="cuda", generator=g).bfloat16()
                part = torch.empty(F.decode_partials(S, H, Tmax), device="cuda")
                cases = [(p, 2.0) for p in (0, 63, 64, 65, Tmax - 1)]
                if S == 3:
                    cases.append((Tmax - 1, 8.0))                 # large q, one planted key: one chunk dominates
                for p, qs in cases:
                    qkv = (torch.randn(S, 3 * C, device="cuda", generator=g) * qs).bfloat16()
                    if qs > 2.0:
                        cache[:, min(p, 130), 0] = qkv[:, :C].view(S, H, 64)
                    pos = torch.tensor([p, 0], dtype=torch.int32, device="cuda")
                    part.fill_(float("nan"))                      # a partial read past chunk pos // 64 shows
                    before = cache.clone()
                    out = torch.empty(S, C, device="cuda").bfloat16()
                    F.attention_decode(qkv, cache, pos, out, part, H)
                    torch.cuda.synchronize()
                    tag = f"attention_decode H={H} Tmax={Tmax} S={S} pos={p}" + (" large q" if qs > 2 else "")
                    assert torch.equal(cache[:, p, 0].reshape(S, C), qkv[:, C:2 * C]), tag
                    assert torch.equal(cache[:, p, 1].reshape(S, C), qkv[:, 2 * C:]), tag
                    keep = torch.ones(Tmax, dtype=torch.bool, device="cuda")
                    keep[p] = False
                    assert torch.equal(cache[:, keep], before[:, keep]), f"{tag}: wrote outside position pos"
                    assert pos.tolist() == [p, 0], f"{tag}: moved pos"
                    ref = _attention_reference(qkv, before, p, H)
                    ok &= _check(tag, out, ref.float(), 2e-2, atol_scale=5e-2)
                del cache, part
    assert ok
    print("attention_decode at every GPT-2 size ok")


GPT2_WIDTHS = {"small": 768, "medium": 1024, "large": 1280, "xl": 1600}


def gpu_embedding_decode_exact():
    from trainingjob_operator_b200.ops import functional as F

    V, L = 50257, 1024
    for name, C in GPT2_WIDTHS.items():
        g = torch.Generator(device="cuda").manual_seed(C)
        wte = torch.randn(V, C, device="cuda", generator=g).bfloat16()
        wpe = (torch.randn(L, C, device="cuda", generator=g) * 0.1).bfloat16()
        tok = torch.tensor([0, V - 1, 12345, 0, V - 1], device="cuda")
        S = tok.numel()
        for p in (0, L - 1):
            buf = torch.full((S + 3, C), 7.0, device="cuda").bfloat16()
            pos = torch.tensor([p, 0], dtype=torch.int32, device="cuda")
            F.embedding_decode(tok, wte, wpe, pos, buf[:S])
            torch.cuda.synchronize()
            want = (wte[tok].float() + wpe[p].float()).bfloat16()
            assert torch.equal(buf[:S].view(torch.int16), want.view(torch.int16)), (name, p)
            assert bool((buf[S:] == 7.0).all()), f"{name} pos={p}: rows after S were written"
            assert pos.tolist() == [p, 0]
    print("embedding_decode exact at every GPT-2 width")


def gpu_decode_gemms():
    """The GEMMs of ``GPT2Generator._step`` (block_n 128) at decode row counts: qkv + bias, proj + bias + residual, fc +
    bias + GELU with the pre-activation saved, fc2 + bias + residual, and the plain logits GEMM over the padded
    vocabulary, against fp64.  Every output, aux and residual is the first M rows of a buffer with a sentinel below."""
    from trainingjob_operator_b200.ops import functional as F
    from trainingjob_operator_b200.ops.selfcheck import _check

    sentinel = 7.0
    ok = True
    for name, C in GPT2_WIDTHS.items():
        g = torch.Generator(device="cuda").manual_seed(C)

        def rnd(*shape, scale=1.0):
            return (torch.randn(*shape, device="cuda", generator=g) * scale).bfloat16()

        shapes = {"qkv": (3 * C, C), "proj": (C, C), "fc": (4 * C, C), "fc2": (C, 4 * C), "logits": (50304, C)}
        W = {k: rnd(n, kk, scale=kk ** -0.5) for k, (n, kk) in shapes.items()}
        bias = {k: rnd(n, scale=0.5) for k, (n, _) in shapes.items()}
        for M in (1, 3, 8, 16, 65):
            for gname, (N, K) in shapes.items():
                x = rnd(M, K)

                def view(init=None, cols=N):
                    buf = torch.full((M + 5, cols), sentinel, device="cuda").bfloat16()
                    if init is not None:
                        buf[:M] = init
                    return buf, buf[:M]

                obuf, out = view()
                kw, pre_ref = {}, None
                ref = x.double() @ W[gname].double().t()
                if gname != "logits":
                    kw["bias"] = bias[gname]
                    ref = ref + bias[gname].double()
                rbuf = abuf = None
                if gname in ("proj", "fc2"):
                    rbuf, kw["residual"] = view(rnd(M, N))
                    rsave = rbuf.clone()
                    ref = ref + kw["residual"].double()
                if gname == "fc":
                    abuf, kw["aux"] = view()
                    kw.update(gelu=True, save_pre=True)
                    pre_ref = ref
                    ref = 0.5 * ref * (1 + torch.tanh(math.sqrt(2 / math.pi) * (ref + 0.044715 * ref ** 3)))
                F.gemm(x, W[gname], out, block_n=128, **kw)
                torch.cuda.synchronize()
                tag = f"{name} {gname} M={M} N={N} K={K}"
                ok &= _check(tag, out, ref.float(), 1e-2)
                if pre_ref is not None:
                    ok &= _check(tag + " pre-activation", kw["aux"], pre_ref.float(), 1e-2)
                    assert bool((abuf[M:] == sentinel).all()), f"{tag}: aux written past row M"
                assert bool((obuf[M:] == sentinel).all()), f"{tag}: output written past row M"
                if rbuf is not None:
                    assert torch.equal(rbuf, rsave), f"{tag}: residual buffer changed"
    assert ok
    print("decode GEMMs ok")


@pytest.mark.gpu
def test_sample_tokens_draw_by_draw_against_the_fp64_oracle():
    _run_case("gpu_sample_tokens_oracle")


@pytest.mark.gpu
def test_sample_tokens_contracts():
    _run_case("gpu_sample_tokens_contracts")


@pytest.mark.gpu
def test_sample_tokens_keeps_negative_zero_ties_and_claims_every_target():
    _run_case("gpu_sample_tokens_regressions")


@pytest.mark.gpu
def test_attention_decode_at_every_gpt2_size_against_fp64():
    _run_case("gpu_attention_decode_sizes")


@pytest.mark.gpu
def test_embedding_decode_is_exact():
    _run_case("gpu_embedding_decode_exact")


@pytest.mark.gpu
def test_decode_gemms_against_fp64_inside_their_rows():
    _run_case("gpu_decode_gemms")


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    globals()[sys.argv[1]]()
