"""HellaSwag for GPT-2 workers: llm.c's eval file, and its completions packed as documents into micro-batches.

The file is what llm.c's ``dev/data/hellaswag.py`` writes (``write_evalfile``): a header of 256 little-endian int32
(magic 20240522, version 1, the number of examples, the longest example in bytes), then one uint16 stream per example:
65535, the example's length in bytes (of the whole stream from the 65535 on), its index, its label, the number of
completions, ``n_ctx`` and the context's tokens, and for each completion ``n_end`` and the ending's tokens.

Each completion ``ctx + end_c`` is scored alone, from position 0: its score is the mean NLL of its ``n_end`` ending
tokens, and the prediction is the completion with the lowest score (the first on a tie), as llm.c reports it.

Instead of one completion per row, the completions are packed into the rows of ``B x T`` micro-batches as documents:
a completion takes ``n_ctx + n_end - 1`` consecutive positions of one row (its tokens but the last as inputs, the next
token as the target of the ``n_end`` positions that predict an ending token, -1 elsewhere), and ``doc_start`` is its
first position.  Padding holds token 0, target -1 and its own position as ``doc_start``, so ``doc_start`` never
decreases along a row.  An example's four completions go in file order, each at the first free position of the current
row or else of the next; an example never straddles two micro-batches.  The micro-batches therefore depend only on the
file, B and T -- never on the world size -- and are assigned to the ranks as the held-out evaluation's are.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Tuple

import numpy as np
import torch

from .data import DataError

MAGIC, VERSION = 20240522, 1
HEADER_INTS = 256
START = 65535
CHOICES = 4


@dataclass
class Example:
    index: int                   # the example's place in the file
    label: int
    ctx: np.ndarray              # int64 context tokens
    ends: List[np.ndarray]       # int64 ending tokens, one array per completion


def read_examples(path: str, vocab: int, seq: int) -> List[Example]:
    """The examples of llm.c's eval file ``path``; ``DataError`` (naming the file, and the example where there is one)
    for anything that is not a well-formed file of 4-completion examples whose tokens are below ``vocab`` and whose
    completions fit in ``seq`` input positions."""
    try:
        raw = open(path, "rb").read()
    except OSError as e:
        raise DataError(f"{path}: cannot read the HellaSwag file: {e}") from None
    if len(raw) < HEADER_INTS * 4:
        raise DataError(f"{path}: truncated file: {len(raw)} bytes, shorter than the {HEADER_INTS * 4}-byte header")
    head = np.frombuffer(raw, dtype="<i4", count=HEADER_INTS)
    if int(head[0]) != MAGIC:
        raise DataError(f"{path}: magic {int(head[0])} is not llm.c's eval file magic {MAGIC}")
    if int(head[1]) != VERSION:
        raise DataError(f"{path}: version {int(head[1])} is not {VERSION}")
    n = int(head[2])
    body = raw[HEADER_INTS * 4:]
    if len(body) % 2:
        raise DataError(f"{path}: truncated file: an odd number of bytes after the header")
    data = np.frombuffer(body, dtype="<u2").astype(np.int64)
    out: List[Example] = []
    pos = 0
    for i in range(n):
        where = f"{path}: example {i}"
        if pos == len(data):
            raise DataError(f"{path}: the header counts {n} examples, the file holds {i}")
        if data[pos] != START:
            raise DataError(f"{where}: missing start delimiter {START} (found {int(data[pos])})")
        if pos + 1 >= len(data):
            raise DataError(f"{where}: truncated file")
        nbytes = int(data[pos + 1])
        if nbytes % 2 or nbytes < 12:
            raise DataError(f"{where}: byte count {nbytes} does not match the example")
        end = pos + nbytes // 2
        if end > len(data):
            raise DataError(f"{where}: truncated file: the example's {nbytes} bytes run past the end")
        s = data[pos:end]

        def field(k: int, what: str) -> int:
            if k >= len(s):
                raise DataError(f"{where}: byte count {nbytes} does not match the example (it ends inside {what})")
            return int(s[k])

        label, ncomp, n_ctx = field(3, "the label"), field(4, "the completion count"), field(5, "the context length")
        if ncomp != CHOICES:
            raise DataError(f"{where}: {ncomp} completions, not {CHOICES}")
        if label >= CHOICES:
            raise DataError(f"{where}: label {label} is not below {CHOICES}")
        if n_ctx == 0:
            raise DataError(f"{where}: empty context")
        k = 6 + n_ctx
        field(k - 1, "the context")
        ctx = s[6:k]
        ends = []
        for c in range(CHOICES):
            n_end = field(k, f"ending {c}")
            if n_end == 0:
                raise DataError(f"{where}: ending {c} is empty")
            field(k + n_end, f"ending {c}")
            ends.append(s[k + 1:k + 1 + n_end])
            k += 1 + n_end
        if k != len(s):
            raise DataError(f"{where}: byte count {nbytes} does not match the example ({k * 2} bytes of fields)")
        for t in (ctx, *ends):
            bad = t[t >= vocab]
            if bad.size:
                raise DataError(f"{where}: token id {int(bad[0])} is outside the vocabulary (size {vocab})")
        for c, e in enumerate(ends):
            if n_ctx + len(e) - 1 > seq:
                raise DataError(f"{where}: completion {c} takes {n_ctx + len(e) - 1} input positions, more than "
                                f"--seq {seq}")
        out.append(Example(i, label, ctx, ends))
        pos = end
    if pos != len(data):
        raise DataError(f"{path}: the header counts {n} examples, the file holds more")
    return out


def write_examples(path: str, examples) -> str:
    """llm.c's eval file of ``examples`` ((label, ctx tokens, [4 ending token lists]) each), as ``write_evalfile``
    writes it: for test fixtures and synthetic benchmarks."""
    stream: List[int] = []
    longest = 0
    for idx, (label, ctx, ends) in enumerate(examples):
        ex = [START, 0, idx, int(label), len(ends), len(ctx), *map(int, ctx)]
        for e in ends:
            ex += [len(e), *map(int, e)]
        ex[1] = 2 * len(ex)
        longest = max(longest, ex[1])
        stream += ex
    head = np.zeros(HEADER_INTS, dtype="<i4")
    head[:4] = (MAGIC, VERSION, len(examples), longest)
    with open(path, "wb") as f:
        f.write(head.tobytes())
        f.write(np.asarray(stream, dtype="<u2").tobytes())
    return path


def pack(examples: List[Example], B: int, T: int, path: str = "") -> List[List[Tuple[int, int, int]]]:
    """Placement of every completion: per micro-batch, per example, per completion (row, first position), as the module
    docstring describes."""
    micro: List[list] = []
    cur: list = []
    row = col = 0

    def place(r: int, p: int, lens):
        spots = []
        for L in lens:
            if p + L > T:
                r, p = r + 1, 0
            spots.append((r, p))
            p += L
        return spots, r, p

    for ex in examples:
        lens = [len(ex.ctx) + len(e) - 1 for e in ex.ends]
        spots, r, p = place(row, col, lens)
        if r >= B:
            if cur:
                micro.append(cur)
            cur = []
            spots, r, p = place(0, 0, lens)
            if r >= B:
                raise DataError(f"{path}: example {ex.index}: its completions ({lens} positions) do not fit in a "
                                f"micro-batch of {B} rows of {T}")
        cur.append(spots)
        row, col = r, p
    if cur:
        micro.append(cur)
    return micro


class HellaSwagData:
    """The examples of an llm.c HellaSwag file, packed into micro-batches of ``B`` rows of ``T`` positions once, as host
    tensors (pinned when ``pin``): for micro-batch k, ``inputs(k)`` gives (tokens, targets, doc_start, spans, labels) as
    ``GPT2Engine.score_forward`` takes them."""

    def __init__(self, path: str, vocab: int, B: int, T: int, pin: bool = False):
        self.path, self.B, self.T = path, B, T
        examples = read_examples(path, vocab, T)
        if not examples:
            raise DataError(f"{path}: no examples")
        self.examples = len(examples)
        placement = pack(examples, B, T, path)
        K, M = len(placement), B * T
        tok = np.zeros((K, M), dtype=np.int64)
        tgt = np.full((K, M), -1, dtype=np.int64)
        ds = np.tile(np.arange(T, dtype=np.int32), (K, B))             # padding: its own position
        spans = np.zeros((self.examples, CHOICES, 2), dtype=np.int32)
        labels = np.zeros(self.examples, dtype=np.int32)
        self.first = [0]                                                 # micro-batch k holds examples [first[k], first[k+1])
        filled = 0
        e = 0
        for k, exs in enumerate(placement):
            for spots in exs:
                ex = examples[e]
                labels[e] = ex.label
                for c, (r, p) in enumerate(spots):
                    seq = np.concatenate([ex.ctx, ex.ends[c]])
                    L = len(seq) - 1
                    a = r * T + p
                    tok[k, a:a + L] = seq[:-1]
                    n_ctx, n_end = len(ex.ctx), len(ex.ends[c])
                    tgt[k, a + n_ctx - 1:a + L] = ex.ends[c]
                    ds[k, a:a + L] = p
                    spans[e, c] = (a + n_ctx - 1, n_end)
                    filled += L
                e += 1
            self.first.append(e)
        self.micro_batches = K
        self.fill = filled / (K * M)                   # share of the positions that hold a completion
        t = [torch.from_numpy(x) for x in (tok, tgt, ds, spans, labels)]
        if pin:
            t = [x.pin_memory() for x in t]
        self.tok, self.tgt, self.doc_start, self.spans, self.labels = t

    def inputs(self, k: int):
        """(tokens int64 [B*T], targets int64 [B*T], doc_start int32 [B*T], spans int32 [E, 4, 2], labels int32 [E]) of
        micro-batch k."""
        a, b = self.first[k], self.first[k + 1]
        return self.tok[k], self.tgt[k], self.doc_start[k], self.spans[a:b], self.labels[a:b]

    def plan(self, world: int, rank: int) -> Tuple[int, ...]:
        """The micro-batches of rank ``rank`` of ``world``: r, r + W, ..., as the held-out evaluation assigns them."""
        from .accumulation import micro_batch_plan

        return micro_batch_plan(self.micro_batches * self.B, self.B, world, rank).micro
