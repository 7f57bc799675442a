"""Token-file data source for the GPT-2 workers (``--data``).

A corpus is one or more shards of GPT-2 token ids, read as one stream in sorted path order.  Two file formats:

* llm.c shards: a header of 256 int32 (``[0]`` = 20240520, ``[1]`` = 1, ``[2]`` = number of tokens), then the tokens as
  uint16;
* raw uint16 token files (nanoGPT's ``train.bin``).

Files are memory-mapped, never read whole.  Sample ``i`` is the window of T+1 tokens starting at token ``i*T`` of the
stream, modulo the number of whole windows (wrapping around starts the next epoch): ``tok`` is its first T tokens and
``tgt`` its last T.  With ``doc_mask`` a sample also has ``doc_start``: position t of the window starts a document when
t == 0 or ``tok[t]`` is the end-of-text token, which thus opens the document it precedes (as in llm.c's shards), and
``doc_start[t]`` is the start of the document holding t.

Every window is checked on the host before it is staged: a token id ``>= vocab_size`` is an error naming the shard and
the offset, so an out-of-range id never reaches the embedding kernel, which indexes the embedding table with it.
"""
from __future__ import annotations

import glob
import os
from typing import List, Optional, Tuple

import numpy as np
import torch

LLMC_MAGIC = 20240520
LLMC_VERSION = 1
LLMC_HEADER_INTS = 256
GPT2_EOT = 50256


class DataError(ValueError):
    pass


def _open_shard(path: str, fmt: str) -> np.ndarray:
    """The tokens of one file as a read-only uint16 memory map.  ``fmt``: "llmc", "raw" or "auto" (llm.c when the file
    starts with llm.c's magic number, raw otherwise)."""
    size = os.path.getsize(path)
    head = np.fromfile(path, dtype="<i4", count=min(LLMC_HEADER_INTS, size // 4))
    is_llmc = fmt == "llmc" or (fmt == "auto" and head.size >= 1 and int(head[0]) == LLMC_MAGIC)
    if is_llmc:
        hdr_bytes = LLMC_HEADER_INTS * 4
        if head.size < LLMC_HEADER_INTS or int(head[0]) != LLMC_MAGIC:
            raise DataError(f"{path}: not an llm.c token shard (bad magic "
                            f"{int(head[0]) if head.size else None}, expected {LLMC_MAGIC})")
        if int(head[1]) != LLMC_VERSION:
            raise DataError(f"{path}: unsupported llm.c shard version {int(head[1])} (expected {LLMC_VERSION})")
        n = int(head[2])
        if n < 0 or size != hdr_bytes + 2 * n:
            raise DataError(f"{path}: size {size} bytes does not match the header's {n} tokens "
                            f"({hdr_bytes + 2 * max(n, 0)} bytes expected)")
        return np.memmap(path, dtype="<u2", mode="r", offset=hdr_bytes, shape=(n,)) if n else np.zeros(0, np.uint16)
    if fmt not in ("raw", "auto"):
        raise ValueError(f"unknown token file format {fmt!r}")
    if size % 2:
        raise DataError(f"{path}: a raw uint16 token file cannot have an odd size ({size} bytes)")
    return np.memmap(path, dtype="<u2", mode="r", shape=(size // 2,)) if size else np.zeros(0, np.uint16)


def expand_paths(spec: str) -> List[str]:
    """A path or a glob -> the shard files, sorted."""
    paths = sorted(glob.glob(spec)) if glob.has_magic(spec) else [spec]
    paths = [p for p in paths if os.path.isfile(p)]
    if not paths:
        raise DataError(f"--data {spec!r}: no such file")
    return paths


class TokenStream:
    """The shards of a corpus as one stream of tokens."""

    def __init__(self, spec: str, fmt: str = "auto"):
        self.paths = expand_paths(spec)
        self.shards = [_open_shard(p, fmt) for p in self.paths]
        self.starts = np.cumsum([0] + [len(s) for s in self.shards])
        self.n_tokens = int(self.starts[-1])

    def locate(self, pos: int) -> Tuple[str, int]:
        """Stream position -> (shard path, token offset inside it)."""
        i = int(np.searchsorted(self.starts, pos, side="right")) - 1
        return self.paths[i], pos - int(self.starts[i])

    def read(self, pos: int, n: int, out: np.ndarray) -> None:
        """out[:n] <- tokens [pos, pos + n) of the stream (may span shards)."""
        done = 0
        while done < n:
            path, off = self.locate(pos + done)
            shard = self.shards[self.paths.index(path)]
            k = min(n - done, len(shard) - off)
            out[done:done + k] = shard[off:off + k]
            done += k


def doc_starts(tok: np.ndarray, eot: int) -> np.ndarray:
    """doc_start[t] of one window: the last position s <= t with s == 0 or tok[s] == eot."""
    idx = np.arange(tok.shape[-1], dtype=np.int32)
    starts = np.where(tok == eot, idx, 0).astype(np.int32)
    return np.maximum.accumulate(starts, axis=-1)


class TokenFileData:
    """Batches of consecutive samples of a token corpus, staged in pinned host memory for the engine's input tensors
    (tok, tgt[, doc_start]).

    ``stage(first, B)`` fills a staging slot with samples ``[first, first + B)`` and returns its tensors; the caller
    enqueues their non-blocking copies and then calls ``in_flight()``.  Slots are a ring of two, each with a CUDA event
    recorded behind its copies: a slot is only rewritten once its previous copies have completed."""

    def __init__(self, spec: str, seq: int, vocab_size: int, doc_mask: bool = False, eot: int = GPT2_EOT,
                 pin: bool = True, fmt: str = "auto"):
        if doc_mask and not 0 <= eot < vocab_size:
            raise DataError(f"end-of-text token {eot} is outside the vocabulary (size {vocab_size})")
        self.stream = TokenStream(spec, fmt)
        self.T, self.vocab, self.doc_mask, self.eot = seq, vocab_size, doc_mask, eot
        self.n_windows = (self.stream.n_tokens - 1) // seq
        if self.n_windows < 1:
            raise DataError(f"--data {spec!r}: {self.stream.n_tokens} tokens do not make one window of {seq + 1}")
        self.pin = pin and torch.cuda.is_available()
        self._slots: List[Optional[dict]] = [None, None]
        self._next = 0
        self._last: Optional[dict] = None
        self.bytes_per_sample = seq * (8 + 8 + (4 if doc_mask else 0))
        self.samples_read: List[int] = []       # sample indices of the last stage() (what this rank trained on)

    def window(self, sample: int) -> np.ndarray:
        """The T+1 tokens of sample ``sample``, checked against the vocabulary."""
        T = self.T
        start = (sample % self.n_windows) * T
        buf = np.empty(T + 1, dtype=np.uint16)
        self.stream.read(start, T + 1, buf)
        bad = np.flatnonzero(buf >= self.vocab)
        if bad.size:
            path, off = self.stream.locate(start + int(bad[0]))
            raise DataError(f"{path}: token id {int(buf[bad[0]])} at token offset {off} is outside the vocabulary "
                            f"(size {self.vocab})")
        return buf

    def sample(self, sample: int):
        """(tok, tgt, doc_start or None) of one sample as numpy arrays (int64, int64, int32)."""
        w = self.window(sample).astype(np.int64)
        tok, tgt = w[:-1], w[1:]
        return tok, tgt, (doc_starts(tok, self.eot) if self.doc_mask else None)

    def _slot(self, B: int) -> dict:
        k = self._next
        self._next ^= 1
        s = self._slots[k]
        if s is None or s["B"] != B:
            n = B * self.T
            s = {"B": B, "event": None, "tok": torch.empty(n, dtype=torch.int64, pin_memory=self.pin),
                 "tgt": torch.empty(n, dtype=torch.int64, pin_memory=self.pin),
                 "doc": torch.empty(n, dtype=torch.int32, pin_memory=self.pin) if self.doc_mask else None}
            self._slots[k] = s
        if s["event"] is not None:
            s["event"].synchronize()            # the copies that last read this slot have completed
            s["event"] = None
        return s

    def stage(self, first: int, B: int, count: Optional[int] = None) -> List[torch.Tensor]:
        """Samples [first, first + B) -> pinned (tok, tgt[, doc_start]) of B*T elements each.  ``count`` < B: only
        samples [first, first + count) are read, and the rows of the others carry token 0 and target -1 (no loss)."""
        T = self.T
        count = B if count is None else count
        toks = np.zeros((B, T + 1), dtype=np.uint16)
        for b in range(count):
            toks[b] = self.window(first + b)         # validated before anything is staged
        s = self._slot(B)
        w = toks.astype(np.int64)
        s["tok"].numpy().reshape(B, T)[:] = w[:, :-1]
        s["tgt"].numpy().reshape(B, T)[:] = w[:, 1:]
        s["tgt"].numpy().reshape(B, T)[count:] = -1
        out = [s["tok"], s["tgt"]]
        if self.doc_mask:
            s["doc"].numpy().reshape(B, T)[:] = doc_starts(w[:, :-1], self.eot)
            out.append(s["doc"])
        self._last = s
        self.samples_read = list(range(first, first + count))
        return out

    def in_flight(self) -> None:
        """The copies of the last staged slot have been enqueued on the current stream."""
        if self.pin and self._last is not None:
            ev = torch.cuda.Event()
            ev.record()
            self._last["event"] = ev
