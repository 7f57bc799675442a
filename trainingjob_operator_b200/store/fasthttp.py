"""Lean HTTP/1.1 header handling for the API server and its client.

``http.server`` and ``http.client`` parse every header block with the e-mail package (``email.feedparser``, policy
objects, ``Message``): ~100 us per message in this interpreter, on both ends of every API call -- more than a third of the
API-server process' CPU time under the throughput benchmark (``tools/throughput_bench.py --daemons``), where that
process is the bottleneck of the three-daemon topology.  The headers this API needs are a handful of ``Name: value``
lines; ``read_headers`` reads them into a case-insensitive dict, ``FastResponse`` is ``http.client.HTTPResponse`` with that
parser, and the server's handler uses it in its own ``parse_request`` (``store/http.py``).  Semantics kept: header names
are case-insensitive, repeated headers are joined with ``", "``, obsolete line folding continues the previous value,
over-long lines / too many headers raise the same ``http.client`` exceptions.

The reference talks to a real kube-apiserver through client-go's REST client
(/root/reference/pkg/client/clientset/versioned/typed/aitrainingjob/v1/aitrainingjob.go:66-190); this is the wire layer
of the single-box replacement.
"""
from __future__ import annotations

import http.client
from typing import Iterator, List, Optional, Tuple

_MAXLINE = 65536
_MAXHEADERS = 100


class Headers(dict):
    """One message's header block: keys are lower-cased names; look-ups are case-insensitive."""

    def get(self, name, default=None):  # type: ignore[override]
        return dict.get(self, name.lower(), default)

    def __getitem__(self, name):
        return dict.__getitem__(self, name.lower())

    def __contains__(self, name) -> bool:  # type: ignore[override]
        return dict.__contains__(self, name.lower())

    def get_all(self, name, default=None) -> Optional[List[str]]:
        v = dict.get(self, name.lower())
        return default if v is None else [v]

    def items(self) -> Iterator[Tuple[str, str]]:  # type: ignore[override]
        return iter(dict.items(self))


def read_headers(fp) -> Headers:
    """Read ``Name: value`` lines up to the blank line that ends the header block."""
    h = Headers()
    last = None
    n = 0
    while True:
        line = fp.readline(_MAXLINE + 1)
        if len(line) > _MAXLINE:
            raise http.client.LineTooLong("header line")
        if line in (b"\r\n", b"\n", b""):
            return h
        n += 1
        if n > _MAXHEADERS:
            raise http.client.HTTPException(f"got more than {_MAXHEADERS} headers")
        if line[:1] in (b" ", b"\t") and last is not None:       # obsolete folding: continuation of the previous value
            dict.__setitem__(h, last, dict.__getitem__(h, last) + " " + line.decode("iso-8859-1").strip())
            continue
        name, sep, value = line.partition(b":")
        if not sep:
            continue                                              # not a header line: ignored, as the e-mail parser does
        last = name.decode("iso-8859-1").strip().lower()
        v = value.decode("iso-8859-1").strip()
        if dict.__contains__(h, last):
            v = dict.__getitem__(h, last) + ", " + v
        dict.__setitem__(h, last, v)


class FastResponse(http.client.HTTPResponse):
    """``HTTPResponse`` whose ``begin`` uses ``read_headers``; status line, chunked / Content-Length / keep-alive
    decisions are the parent's, statement for statement in effect."""

    def begin(self) -> None:
        if self.headers is not None:
            return
        while True:
            version, status, reason = self._read_status()
            if status != http.client.CONTINUE:
                break
            read_headers(self.fp)                                 # the header block of the 100 response
        self.code = self.status = status
        self.reason = reason.strip()
        if version in ("HTTP/1.0", "HTTP/0.9"):
            self.version = 10
        elif version.startswith("HTTP/1."):
            self.version = 11
        else:
            raise http.client.UnknownProtocol(version)
        self.headers = self.msg = read_headers(self.fp)
        tr_enc = self.headers.get("transfer-encoding")
        if tr_enc and tr_enc.lower() == "chunked":
            self.chunked = True
            self.chunk_left = None
        else:
            self.chunked = False
        self.will_close = self._check_close()
        self.length = None
        length = self.headers.get("content-length")
        if length and not self.chunked:
            try:
                self.length = int(length)
            except ValueError:
                self.length = None
            else:
                if self.length < 0:
                    self.length = None
        if status in (http.client.NO_CONTENT, http.client.NOT_MODIFIED) or 100 <= status < 200 or self._method == "HEAD":
            self.length = 0
        if not self.will_close and not self.chunked and self.length is None:
            self.will_close = True
