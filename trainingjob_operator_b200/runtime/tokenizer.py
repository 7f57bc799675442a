"""Token-id-to-text decoding with an llm.c ``gpt2_tokenizer.bin``.

The file is a header of 256 uint32 -- magic 20240328, version (1 or 2), vocabulary size, and for version 2 the
end-of-text id -- followed by one record per token: a uint8 length and that many bytes.  Decoding only: there is no
BPE encoder, so prompts are given as token ids.
"""
from __future__ import annotations

import struct
from typing import Iterable, List, Optional

MAGIC = 20240328


class TokenizerError(ValueError):
    pass


class Tokenizer:
    def __init__(self, path: str):
        self.path = path
        try:
            with open(path, "rb") as f:
                raw = f.read()
        except OSError as e:
            raise TokenizerError(f"{path}: cannot read the tokenizer: {e}") from None
        if len(raw) < 256 * 4:
            raise TokenizerError(f"{path}: truncated header ({len(raw)} bytes, a tokenizer starts with 1024)")
        header = struct.unpack("<256I", raw[:1024])
        if header[0] != MAGIC:
            raise TokenizerError(f"{path}: bad magic {header[0]} (an llm.c tokenizer has {MAGIC})")
        if header[1] not in (1, 2):
            raise TokenizerError(f"{path}: unknown tokenizer version {header[1]} (1 or 2 are known)")
        self.version, n = header[1], header[2]
        self.eot: Optional[int] = header[3] if self.version == 2 else None
        self.tokens: List[bytes] = []
        off = 1024
        for i in range(n):
            if off >= len(raw):
                raise TokenizerError(f"{path}: truncated at token {i} of {n}")
            length = raw[off]
            if off + 1 + length > len(raw):
                raise TokenizerError(f"{path}: truncated at token {i} of {n}")
            self.tokens.append(raw[off + 1:off + 1 + length])
            off += 1 + length

    @property
    def vocab_size(self) -> int:
        return len(self.tokens)

    def decode_bytes(self, ids: Iterable[int]) -> bytes:
        out = []
        for t in ids:
            t = int(t)
            if not 0 <= t < len(self.tokens):
                raise ValueError(f"token id {t} is outside the tokenizer {self.path} ({len(self.tokens)} tokens)")
            out.append(self.tokens[t])
        return b"".join(out)

    def decode(self, ids: Iterable[int]) -> str:
        """Text of the ids; bytes that are not UTF-8 (a token can end inside a character) become U+FFFD."""
        return self.decode_bytes(ids).decode("utf-8", errors="replace")
