"""Plain-PyTorch stand-ins for the entry points of ``trainingjob_operator_b200.ops.functional`` -- TEST ONLY.

The engines (``models/gpt2.py``, ``models/bert.py``), the trainer and the worker adapters only run on a GPU box, where
they call hand-written sm_90a kernels; nothing of that can execute without a GPU.  ``install()`` replaces the
kernel entry points by functions with the same contracts (same arguments, same in-place outputs, same accumulate /
overwrite rules, bf16 storage with fp32 math) so that the *control flow around the kernels* -- buffer rotation, which
gradient goes where, bucket hooks, optimizer arguments, the per-GEMM kernel table, the side-stream bookkeeping -- runs
on CPU and is checked against the fp32 reference models on every commit.  It says nothing about the kernels themselves;
those are checked on the device by ``ops/selfcheck.py`` (``tests/test_gpu_kernels.py``).

Every stand-in first applies the host-side refusals of its library function (``REFUSALS``): a call the library answers
with an error code raises ``lib.KernelError`` with that code here too, so an engine change that the kernels would refuse
fails on the CPU as well.  ``tests/test_kernel_contracts.py`` holds the table to the library's ``return -N`` sites.

Never imported by the package: on a GPU box a missing kernel library raises (``ops/lib.py``), there is no fallback.
"""
from __future__ import annotations

import functools
import math
import re
import threading
from types import SimpleNamespace

import torch
import torch.nn.functional as TF

from trainingjob_operator_b200.ops import functional as F
from trainingjob_operator_b200.ops.functional import gemm_epilogue, xent_blocks   # host arithmetic; not recorded as launches
from trainingjob_operator_b200.ops.lib import KernelError

CALLS = {"n": 0, "gemm_block_n": []}
XENT_CALLS = []       # block_n of every gemm_xent call
_K0, _K1 = math.sqrt(2.0 / math.pi), 0.044715


# ------------------------------------------------------------------------------------ the library's refusals
# gemm_bf16_wgmma_kernel<kBN, kAMN, kBMN, kCM, kEpi>, mangled: the name of every compiled GEMM instantiation
GEMM_KERNEL_NAME = re.compile(r"gemm_bf16_wgmma_kernelILi(\d+)ELb([01])ELb([01])ELi(\d+)ELi(\d+)E")


def gemm_kernel_keys(names):
    """(block_n, a_mn, b_mn, cluster size, epilogue bits) of each GEMM instantiation among ``names``."""
    out = set()
    for name in names:
        m = GEMM_KERNEL_NAME.search(name)
        if m:
            bn, amn, bmn, cm, epi = (int(g) for g in m.groups())
            out.add((bn, bool(amn), bool(bmn), cm, epi))
    return out


@functools.lru_cache(maxsize=None)
def compiled_gemm_kernels():
    """The GEMM instantiations of the built library: its host code registers every kernel by its mangled name."""
    F.lib.load()                                     # builds the library when it is missing
    blob = F.lib.LIB_PATH.read_bytes().decode("latin-1")
    return frozenset(gemm_kernel_keys(m.group(0) for m in GEMM_KERNEL_NAME.finditer(blob)))


def gemm_kernel_key(c):
    """The instantiation ``aitj_gemm_bf16`` looks up for the call ``c``: its tile choice, and its epilogue as keyed in
    kGemmKernels (column sums, the cross-entropy's fp32 keying, the owner-sharded split that moves afterwards)."""
    cm = 4 if c.block_n == 1024 else (2 if c.block_n == 512 else 1)
    bn = 256 if cm > 1 else (c.block_n or (256 if c.N > 128 else 128))
    kb = -(-c.K // 64)
    split = min(max(c.split_k, 1), kb)
    per = -(-kb // split)
    split = -(-kb // per)
    epi = (c.flags & ~F.EPI_COLSUM) | (F.EPI_COLSUM if c.colsum else 0)
    if epi & F.EPI_XENT:
        epi |= F.EPI_OUT_F32
    if epi & F.EPI_PEER and split > 1:
        epi &= ~F.EPI_PEER
    return bn, bool(c.a_mn), bool(c.b_mn), cm, epi


def _nonempty(c):
    return c.M > 0 and c.N > 0 and c.K > 0          # an empty GEMM returns 0 before the checks below


def _heads(c):
    return c.B > 0 and c.T > 0 and c.H > 0          # an empty attention returns 0 before its checks


def _xent_bad(c):
    if c.flags & F.EPI_XENT:
        return (c.flags != F.EPI_XENT or c.split_k > 1 or not (c.xent_target and c.xent_part and c.xent_tgt)
                or not 1 <= c.vocab <= c.N or c.xent_part % 8)
    return bool(c.xent_target)


_LN_FWD_C = (256, 512, 768, 1024, 1536, 2048)

# (library function, error code) -> (reason, predicate over the call's arguments, named as in the C signature; pointers
# are integer addresses, 0 for null).  Rows of one function are in the order the library tests them.
REFUSALS = {
    ("aitj_gemm_bf16", -8): ("EPI_XENT with another bit, a split, a missing buffer, vocab outside [1, N] or partials "
                             "not 8-byte aligned; or cross-entropy buffers given to another GEMM", _xent_bad),
    ("aitj_gemm_bf16", -1): ("N, lda, ldb or ldc is not a multiple of 8",
                             lambda c: _nonempty(c) and bool(c.N % 8 or c.lda % 8 or c.ldb % 8 or c.ldc % 8)),
    ("aitj_gemm_bf16", -4): ("out, or the aux / residual the epilogue reads, is not 16-byte aligned (TMA)",
                             lambda c: _nonempty(c) and bool(c.out % 16 or (c.flags & (F.EPI_SAVE_PRE | F.EPI_DGELU)
                                                                          and c.aux % 16)
                                                             or (c.flags & F.EPI_RESIDUAL and c.residual % 16))),
    ("aitj_gemm_bf16", -2): ("split-K without EPI_ACCUM",
                             lambda c: _nonempty(c) and c.split_k > 1 and not c.flags & F.EPI_ACCUM),
    ("aitj_gemm_bf16", -5): ("multicast or owner-sharded output without EPI_ACCUM",
                             lambda c: _nonempty(c) and bool(c.flags & (F.EPI_MC | F.EPI_PEER))
                             and not c.flags & F.EPI_ACCUM),
    ("aitj_gemm_bf16", -3): ("block_n is not 0, 128, 256, 512 or 1024",
                             lambda c: _nonempty(c) and c.block_n not in (0, 128, 256, 512, 1024)),
    ("aitj_gemm_bf16", -6): ("column sums of an fp32 output",
                             lambda c: _nonempty(c) and bool(c.colsum)
                             and bool(c.flags & (F.EPI_OUT_F32 | F.EPI_ACCUM | F.EPI_XENT))),
    ("aitj_gemm_bf16", -7): ("no kernel is compiled for this operand layout, epilogue and tile",
                             lambda c: _nonempty(c) and gemm_kernel_key(c) not in compiled_gemm_kernels()),
    ("aitj_gemm_set_peers", -1): ("a peer table of fewer than 1 or more than 8 ranks", lambda c: not 1 <= c.n <= 8),
    ("aitj_attn_fwd", -1): ("T is not a multiple of 128", lambda c: _heads(c) and c.T % 128 != 0),
    ("aitj_attn_fwd", -5): ("a document mask without causal attention",
                            lambda c: _heads(c) and bool(c.doc_start) and not c.causal),
    ("aitj_attn_fwd", -4): ("doc_start not 8-byte aligned, or qkv / out not 16-byte aligned",
                            lambda c: _heads(c) and bool(c.doc_start % 8 or c.qkv % 16 or c.out % 16)),
    ("aitj_attn_bwd", -1): ("T is not a multiple of 128", lambda c: _heads(c) and c.T % 128 != 0),
    ("aitj_attn_bwd", -5): ("a document mask without causal attention",
                            lambda c: _heads(c) and bool(c.doc_start) and not c.causal),
    ("aitj_attn_bwd", -4): ("doc_start not 8-byte aligned, or qkv / d_out not 16-byte aligned",
                            lambda c: _heads(c) and bool(c.doc_start % 8 or c.qkv % 16 or c.d_out % 16)),
    ("aitj_layernorm_fwd", -1): ("C is not 256, 512, 768, 1024, 1536 or 2048", lambda c: c.C not in _LN_FWD_C),
    ("aitj_layernorm_bwd", -1): ("C is not 256, 512, 768 or 1024", lambda c: c.C not in _LN_FWD_C[:4]),
    ("aitj_embedding_fwd", -1): ("C is not a multiple of 8", lambda c: c.C % 8 != 0),
    ("aitj_embedding_bwd", -1): ("C is not a multiple of 4", lambda c: c.C % 4 != 0),
    ("aitj_embedding3_fwd", -1): ("C is not a multiple of 8", lambda c: c.C % 8 != 0),
    ("aitj_embedding3_bwd", -1): ("C is not a multiple of 4", lambda c: c.C % 4 != 0),
    ("aitj_softmax_xent", -1): ("Vp is not a multiple of 8, or V > Vp", lambda c: c.Vp % 8 != 0 or c.V > c.Vp),
    ("aitj_softmax_xent", -2): ("a row of Vp > 102400 logits does not fit in shared memory",
                                lambda c: c.Vp * 2 > 200 * 1024),
    ("aitj_xent_finish", -1): ("no column block", lambda c: c.M > 0 and c.nblk < 1),
    ("aitj_colsum", -1): ("N is not a multiple of 8", lambda c: c.N % 8 != 0),
    ("aitj_qkv_gather_colsum", -1): ("D is not a multiple of 8", lambda c: c.D % 8 != 0),
    ("aitj_sumsq", -1): ("n is not a multiple of 4", lambda c: c.n % 4 != 0),
    ("aitj_fused_set_peers", -1): ("a peer table of fewer than 1 or more than 8 ranks", lambda c: not 1 <= c.n <= 8),
    ("aitj_peer_push", -1): ("n is not a multiple of 4", lambda c: c.n % 4 != 0),
    ("aitj_adamw", -1): ("n is not a multiple of 256", lambda c: c.n % 256 != 0),
    ("aitj_mc_push", -1): ("n is not a multiple of 4", lambda c: c.n % 4 != 0),
    ("aitj_cast_f32_bf16", -1): ("n is not a multiple of 4", lambda c: c.n % 4 != 0),
    ("aitj_gelu_fwd", -1): ("n is not a multiple of 8", lambda c: c.n % 8 != 0),
    ("aitj_gelu_bwd", -1): ("n is not a multiple of 8", lambda c: c.n % 8 != 0),
}


def refuse(fn: str, **args) -> None:
    """Raise ``KernelError`` with the code the library function ``fn`` returns for these arguments, if it refuses them."""
    c = SimpleNamespace(**args)
    for (name, code), (_reason, bad) in REFUSALS.items():
        if name == fn and bad(c):
            raise KernelError(f"{fn} failed with code {code}", code)


def _p(t) -> int:
    return 0 if t is None else int(t.data_ptr())


# ------------------------------------------------------------------------------------ owner-sharded mode (peer memory)
# Several "ranks" live in ONE process (FakeShard objects of one FakeWorld).  A kernel that is given a PeerView -- the
# LOCAL address of a gradient inside the symmetric buffer -- adds every piece into the copy of the rank that OWNS it;
# the emulation finds the symmetric buffer by its storage and does the same with slices.
_WORLDS = {}          # storage data_ptr of a rank's symmetric gradient buffer -> (FakeWorld, rank)


class FakeShard:
    """What ``parallel.symm.ShardedGradState`` offers the engine, without symmetric memory."""

    available = True
    reason = ""

    def __init__(self, world: "FakeWorld", rank: int, params):
        from trainingjob_operator_b200.parallel.symm import shard_bounds

        self.fw, self.rank, self.world, self.params = world, rank, world.n, params
        total = params.total
        self.g = torch.zeros(total + 64, dtype=torch.float32)
        self.w = torch.zeros(total, dtype=torch.bfloat16)
        self.bounds = shard_bounds(params.specs, total, self.world)
        self.lo, self.hi = self.bounds[rank], self.bounds[rank + 1]
        self.w_mc = 0                                   # "multicast address" of w: element offset * 2
        self.parts_mc = FakeWorld.PARTS_TOKEN + world.uid
        _WORLDS[self.g.untyped_storage().data_ptr()] = (world, rank)
        self.barriers = 0

    @property
    def parts(self):
        return self.g[self.params.total:self.params.total + self.world]

    def barrier(self):
        """Every rank runs in its own thread: a real barrier, like the device-side one between the ranks' streams."""
        self.barriers += 1
        self.fw.sync.wait(timeout=120)


class FakeWorld:
    PARTS_TOKEN = 1 << 40
    _next = 0

    def __init__(self, n: int):
        refuse("aitj_gemm_set_peers", n=n)          # ShardedGradState installs the peer tables of both libraries
        refuse("aitj_fused_set_peers", n=n)
        self.n = n
        FakeWorld._next += 1
        self.uid = FakeWorld._next
        self.shards = []
        self.sync = threading.Barrier(n)
        _PARTS[FakeWorld.PARTS_TOKEN + self.uid] = self

    def attach(self, params) -> FakeShard:
        sh = FakeShard(self, len(self.shards), params)
        self.shards.append(sh)
        params.attach_shard(sh)
        return sh


_PARTS = {}
_ADD_LOCK = threading.Lock()
_CURRENT = {"world": None}      # the world whose bf16 copies an `adamw(p16_multicast=True)` sweep stores into


def _peer_add(local: torch.Tensor, delta: torch.Tensor) -> None:
    """``local`` (a view into one rank's symmetric gradient buffer) += delta, each element in its OWNER's copy."""
    world, _rank = _WORLDS[local.untyped_storage().data_ptr()]
    assert local.is_contiguous()
    off, n = local.storage_offset(), local.numel()
    flat = delta.reshape(-1).float()
    with _ADD_LOCK:                                   # red.add is atomic; two threads' add_ on one slice are not
        for o, sh in enumerate(world.shards):
            a, b = max(off, sh.bounds[o]), min(off + n, sh.bounds[o + 1])
            if b > a:
                sh.g[a:b].add_(flat[a - off:b - off])


class _PeerSink:
    """Stands in for a PeerView destination inside the emulated kernels: ``add_`` goes to the owners."""

    def __init__(self, pv):
        self.t = pv.t
        self.shape, self.dtype = pv.t.shape, pv.t.dtype

    def add_(self, y):
        _peer_add(self.t, y)
        return self

    def index_add_(self, dim, idx, src):
        tmp = torch.zeros(self.t.shape, dtype=torch.float32)
        tmp.index_add_(dim, idx, src)
        _peer_add(self.t, tmp)
        return self


def _dst(t):
    return _PeerSink(t) if hasattr(t, "is_peer") else t   # PeerView -> adds land in the owning rank's copy


def _gelu_grad(x: torch.Tensor) -> torch.Tensor:
    u = _K0 * (x + _K1 * x ** 3)
    th = torch.tanh(u)
    return 0.5 * (1 + th) + 0.5 * x * (1 - th * th) * _K0 * (1 + 3 * _K1 * x * x)


def num_sms() -> int:
    return 132


def gemm(a, b, out, *, a_mn=False, b_mn=False, bias=None, residual=None, aux=None, gelu=False, dgelu=False,
         save_pre=False, accumulate=False, split_k=1, block_n=0, max_ctas=0, colsum=None):
    CALLS["n"] += 1
    CALLS["gemm_block_n"].append(block_n)
    assert a.dtype == torch.bfloat16 and b.dtype == torch.bfloat16
    assert a.dim() == 2 and b.dim() == 2 and a.stride(1) == 1 and b.stride(1) == 1 and out.stride(1) == 1
    A = a.float().t() if a_mn else a.float()
    Bm = b.float() if b_mn else b.float().t()
    assert A.shape[1] == Bm.shape[0], (a.shape, b.shape, a_mn, b_mn)
    o = _dst(out)
    assert tuple(o.shape) == (A.shape[0], Bm.shape[1]), (o.shape, A.shape, Bm.shape)
    flags = gemm_epilogue(out, bias=bias, residual=residual, aux=aux, gelu=gelu, dgelu=dgelu, save_pre=save_pre,
                          accumulate=accumulate, colsum=colsum)
    refuse("aitj_gemm_bf16", A=_p(a), B=_p(b), out=_p(out), M=A.shape[0], N=Bm.shape[1], K=A.shape[1],
           lda=a.stride(0), ldb=b.stride(0), ldc=out.stride(0), a_mn=int(a_mn), b_mn=int(b_mn), bias=_p(bias),
           residual=_p(residual), aux=_p(aux), flags=flags & ~F.EPI_COLSUM, split_k=int(split_k), block_n=int(block_n),
           max_ctas=int(max_ctas), colsum=_p(colsum), xent_target=0, xent_part=0, xent_tgt=0, vocab=0)
    y = A @ Bm
    if bias is not None:
        y = y + bias.float()
    if save_pre:
        aux.copy_(y)
    if gelu:
        y = TF.gelu(y, approximate="tanh")
    if dgelu:
        y = y * _gelu_grad(aux.float())
    if residual is not None:
        y = y + residual.float()
    if accumulate:
        o.add_(y)
    else:
        o.copy_(y)
    if colsum is not None:
        _dst(colsum).add_(o.float().sum(0))
    return out


def layernorm_fwd(x, gamma, beta, y, mean, rstd, eps=1e-5):
    CALLS["n"] += 1
    refuse("aitj_layernorm_fwd", M=x.shape[0], C=x.shape[1])
    xf = x.float()
    mu = xf.mean(1)
    var = xf.var(1, unbiased=False)
    r = torch.rsqrt(var + eps)
    mean.copy_(mu)
    rstd.copy_(r)
    y.copy_((xf - mu[:, None]) * r[:, None] * gamma.float() + beta.float())
    return y


def layernorm_bwd(dy, x, gamma, mean, rstd, dx, dgamma, dbeta, dres=None, dxsum=None):
    CALLS["n"] += 1
    refuse("aitj_layernorm_bwd", M=x.shape[0], C=x.shape[1])
    h = (x.float() - mean[:, None]) * rstd[:, None]
    d = dy.float()
    _dst(dgamma).add_((d * h).sum(0))
    _dst(dbeta).add_(d.sum(0))
    a = d * gamma.float()
    s1 = a.mean(1, keepdim=True)
    s2 = (a * h).mean(1, keepdim=True)
    v = rstd[:, None] * (a - s1 - h * s2)
    if dres is not None:
        v = v + dres.float()
    if dxsum is not None:
        _dst(dxsum).add_(v.sum(0))
    dx.copy_(v)                     # after the reads: dx may alias dres / dy
    return dx


def _pos(M, T, dev):
    return torch.arange(M, device=dev) % T


def embedding_fwd(tok, wte, wpe, out, T):
    CALLS["n"] += 1
    refuse("aitj_embedding_fwd", M=out.shape[0], T=T, C=out.shape[1])
    v = wte[tok].float()
    if wpe is not None:
        v = v + wpe[_pos(tok.numel(), T, tok.device)].float()
    out.copy_(v)
    return out


def embedding_bwd(tok, dx, dwte, dwpe, T):
    CALLS["n"] += 1
    refuse("aitj_embedding_bwd", M=dx.shape[0], T=T, C=dx.shape[1])
    _dst(dwte).index_add_(0, tok, dx.float())
    if dwpe is not None:
        _dst(dwpe).index_add_(0, _pos(tok.numel(), T, tok.device), dx.float())


def embedding3_fwd(tok, typ, wte, wpe, wtt, out, T):
    CALLS["n"] += 1
    refuse("aitj_embedding3_fwd", M=out.shape[0], T=T, C=out.shape[1])
    out.copy_(wte[tok].float() + wpe[_pos(tok.numel(), T, tok.device)].float() + wtt[typ].float())
    return out


def embedding3_bwd(tok, typ, dx, dwte, dwpe, dwtt, T):
    CALLS["n"] += 1
    refuse("aitj_embedding3_bwd", M=dx.shape[0], T=T, C=dx.shape[1])
    d = dx.float()
    _dst(dwte).index_add_(0, tok, d)
    _dst(dwpe).index_add_(0, _pos(tok.numel(), T, tok.device), d)
    _dst(dwtt).index_add_(0, typ, d)


def softmax_xent(logits, target, loss, V, gscale):
    CALLS["n"] += 1
    refuse("aitj_softmax_xent", M=logits.shape[0], V=V, Vp=logits.shape[1])
    z = logits[:, :V].float()
    lse = torch.logsumexp(z, 1)
    valid = (target >= 0) & (target < V)
    t = target.clamp(0, V - 1)
    nll = lse - z.gather(1, t[:, None])[:, 0]
    loss.copy_(torch.where(valid, nll, torch.zeros_like(nll)))
    p = torch.softmax(z, 1)
    p.scatter_add_(1, t[:, None], -torch.ones_like(nll)[:, None])
    p = p * gscale * valid[:, None].float()
    logits.zero_()
    logits[:, :V].copy_(p)


def gemm_xent(x, w, target, vocab, part, tgt_logit, block_n=0):
    """What the EPI_XENT kernel stores: per (row, 128-column block) (max, sum of exp(z - max)) over the columns below
    ``vocab``, and the target's logit, for the rows with a target; the other rows are left as they were."""
    XENT_CALLS.append(block_n)
    assert x.dtype == torch.bfloat16 and w.dtype == torch.bfloat16 and x.stride(1) == 1 and w.stride(1) == 1
    z = x.float() @ w.float().t()
    M, N = z.shape
    nb = xent_blocks(N)
    assert tuple(part.shape) == (M, nb, 2) and 0 < vocab <= N
    refuse("aitj_gemm_bf16", A=_p(x), B=_p(w), out=0, M=M, N=N, K=x.shape[1], lda=x.stride(0), ldb=w.stride(0),
           ldc=0, a_mn=0, b_mn=0, bias=0, residual=0, aux=0, flags=F.EPI_XENT, split_k=1, block_n=int(block_n),
           max_ctas=0, colsum=0, xent_target=_p(target), xent_part=_p(part), xent_tgt=_p(tgt_logit), vocab=int(vocab))
    zp = torch.full((M, nb * 128), float("-inf"), device=z.device)
    zp[:, :vocab] = z[:, :vocab]
    zb = zp.view(M, nb, 128)
    mx = zb.max(2).values
    s = torch.exp(zb - torch.where(torch.isinf(mx), torch.zeros_like(mx), mx)[..., None]).sum(2)
    live = target >= 0
    part[live] = torch.stack([mx, s], 2)[live]
    tgt_logit[live] = z[live].gather(1, target[live][:, None])[:, 0]


def xent_finish(part, tgt_logit, target, loss, acc):
    refuse("aitj_xent_finish", M=part.shape[0], nblk=part.shape[1])
    m, s = part[..., 0], part[..., 1]
    live = target >= 0
    mm = torch.where(s > 0, m, torch.full_like(m, float("-inf"))).max(1).values
    mm = torch.where(live, mm, torch.zeros_like(mm))
    tot = torch.where(s > 0, s * torch.exp(m - mm[:, None]), torch.zeros_like(s)).sum(1)
    nll = torch.where(live, mm + torch.log(tot) - tgt_logit, torch.zeros_like(mm))
    loss.copy_(nll)
    acc[0] += nll.double().sum()
    acc[1] += float(live.sum())


def colsum(dy, db):
    CALLS["n"] += 1
    refuse("aitj_colsum", M=dy.shape[0], N=dy.shape[1])
    _dst(db).add_(dy.float().sum(0))


def _qkv_heads(qkv, B, T, H):
    q5 = qkv.view(B, T, 3, H, 64)
    return (q5[:, :, i].transpose(1, 2).float() for i in range(3))


def _doc_allowed(doc_start, B, T, dev):
    """[B, 1, T, T]: query q sees key k iff doc_start[q] <= k <= q."""
    ds = doc_start.view(B, 1, T, 1).long()
    k = torch.arange(T, device=dev).view(1, 1, 1, T)
    q = torch.arange(T, device=dev).view(1, 1, T, 1)
    return (k >= ds) & (k <= q)


def attention_fwd(qkv, out, lse, B, T, H, causal=True, scale=0.0, doc_start=None):
    CALLS["n"] += 1
    assert qkv.shape == (B * T, 3 * H * 64)
    F._check_doc_start(doc_start, B, T, causal)
    refuse("aitj_attn_fwd", qkv=_p(qkv), out=_p(out), lse=_p(lse), doc_start=_p(doc_start), B=B, T=T, H=H,
           causal=int(causal), scale=float(scale))
    q, k, v = _qkv_heads(qkv, B, T, H)
    s = (q @ k.transpose(-1, -2)) * (scale or 1.0 / 8.0)
    if doc_start is not None:
        s = s.masked_fill(~_doc_allowed(doc_start, B, T, qkv.device), float("-inf"))
    elif causal:
        s = s.masked_fill(torch.ones(T, T, dtype=torch.bool, device=qkv.device).triu(1), float("-inf"))
    lse.view(B, H, T).copy_(torch.logsumexp(s, -1))
    o = torch.softmax(s, -1) @ v
    out.view(B, T, H, 64).copy_(o.transpose(1, 2))
    return out


def attention_bwd(qkv, out, d_out, lse, delta, dq_acc, d_qkv, B, T, H, causal=True, scale=0.0, doc_start=None):
    CALLS["n"] += 1
    F._check_doc_start(doc_start, B, T, causal)
    refuse("aitj_attn_bwd", qkv=_p(qkv), out=_p(out), d_out=_p(d_out), doc_start=_p(doc_start), B=B, T=T, H=H,
           causal=int(causal), scale=float(scale))
    assert float(dq_acc.abs().max()) == 0.0, "dq_acc must be zero on entry"
    q, k, v = (t.requires_grad_(True) for t in _qkv_heads(qkv, B, T, H))
    with torch.enable_grad():
        if doc_start is not None:
            o = TF.scaled_dot_product_attention(q, k, v, attn_mask=_doc_allowed(doc_start, B, T, qkv.device),
                                                scale=(scale or None))
        else:
            o = TF.scaled_dot_product_attention(q, k, v, is_causal=causal, scale=(scale or None))
        gq, gk, gv = torch.autograd.grad(o, (q, k, v), d_out.view(B, T, H, 64).transpose(1, 2).float())
    dst = d_qkv.view(B, T, 3, H, 64)
    for i, g in enumerate((gq, gk, gv)):
        dst[:, :, i].copy_(g.transpose(1, 2))
    return d_qkv


def qkv_gather_colsum(dq, dk, dv, d_qkv, db):
    CALLS["n"] += 1
    B, H, T, D = dq.shape
    for t in (dq, dk, dv):
        if t.stride(3) != 1 or tuple(t.shape) != (B, H, T, D):
            raise ValueError("qkv_gather_colsum: need [B,H,T,D] tensors with unit D stride")
    refuse("aitj_qkv_gather_colsum", B=B, T=T, H=H, D=D)
    dst = d_qkv.view(B, T, 3, H, D)
    for i, g in enumerate((dq, dk, dv)):
        dst[:, :, i].copy_(g.transpose(1, 2))
    _dst(db).add_(d_qkv.float().sum(0))


def sumsq(g, out):
    CALLS["n"] += 1
    refuse("aitj_sumsq", n=g.numel())
    out.add_((g.float() ** 2).sum())


def adamw(p, g, m, v, p16, wd_mask, *, lr, beta1=0.9, beta2=0.95, eps=1e-8, weight_decay=0.1, step=1, sumsq_buf=None,
          max_norm=0.0, grad_div=1.0, zero_grad=True, dyn=None, sumsq_n=1, p16_multicast=False):
    CALLS["n"] += 1
    refuse("aitj_adamw", n=p.numel())
    assert wd_mask.numel() * 256 >= p.numel()      # one weight-decay flag per 256 elements
    bc1, bc2 = 1.0 - beta1 ** step, 1.0 - beta2 ** step
    if dyn is not None:
        lr, bc1, bc2 = float(dyn[0]), float(dyn[1]), float(dyn[2])
    clip = 1.0
    if sumsq_buf is not None and max_norm > 0:
        norm = math.sqrt(float(sumsq_buf[:sumsq_n].sum())) / grad_div
        if norm > max_norm:
            clip = max_norm / (norm + 1e-6)
    gr = g * (clip / grad_div)
    m.mul_(beta1).add_(gr, alpha=1 - beta1)
    v.mul_(beta2).addcmul_(gr, gr, value=1 - beta2)
    wd = wd_mask.to(torch.float32).repeat_interleave(256)[:p.numel()] * weight_decay
    p.sub_(lr * ((m / bc1) / ((v / bc2).sqrt() + eps) + wd * p))
    if zero_grad:
        g.zero_()
    if p16_multicast:
        # `p16` is the multicast address of this range of the bf16 copy: one store lands in every rank's copy
        lo = int(p16) // 2
        for sh in _CURRENT["world"].shards:
            sh.w[lo:lo + p.numel()].copy_(p)
    else:
        p16.copy_(p)


def cast_f32_bf16(src, dst):
    CALLS["n"] += 1
    refuse("aitj_cast_f32_bf16", n=src.numel())
    dst.copy_(src)


def gelu_fwd(x, y):
    CALLS["n"] += 1
    refuse("aitj_gelu_fwd", n=x.numel())
    y.copy_(TF.gelu(x.float(), approximate="tanh"))


def gelu_bwd(x, dy, dx):
    CALLS["n"] += 1
    refuse("aitj_gelu_bwd", n=x.numel())
    dx.copy_(dy.float() * _gelu_grad(x.float()))


def peer_push(dst_local, src):
    CALLS["n"] += 1
    refuse("aitj_peer_push", n=src.numel())
    _peer_add(dst_local, src)
    src.zero_()


def norm_share(parts_mc_ptr, mine, rank):
    CALLS["n"] += 1
    world = _PARTS[int(parts_mc_ptr)]
    for sh in world.shards:
        sh.parts[rank] = float(mine[0])


def mc_push(dst_mc_ptr, src, n):
    refuse("aitj_mc_push", n=int(n))
    raise AssertionError("the multicast all-reduce (mc) path is not emulated")


def install(monkeypatch=None) -> None:
    """Replace the kernel entry points of ``ops.functional`` (via ``monkeypatch`` when given, else permanently -- for
    subprocess scripts)."""
    from trainingjob_operator_b200.ops import functional as F

    table = dict(num_sms=num_sms, gemm=gemm, layernorm_fwd=layernorm_fwd, layernorm_bwd=layernorm_bwd,
                 embedding_fwd=embedding_fwd, embedding_bwd=embedding_bwd, embedding3_fwd=embedding3_fwd,
                 embedding3_bwd=embedding3_bwd, softmax_xent=softmax_xent, colsum=colsum, attention_fwd=attention_fwd,
                 attention_bwd=attention_bwd, qkv_gather_colsum=qkv_gather_colsum, sumsq=sumsq, adamw=adamw,
                 cast_f32_bf16=cast_f32_bf16, gelu_fwd=gelu_fwd, gelu_bwd=gelu_bwd, mc_push=mc_push,
                 peer_push=peer_push, norm_share=norm_share, gemm_xent=gemm_xent, xent_finish=xent_finish)
    # auto_split_k is host-side arithmetic: keep the real one (it asks num_sms(), which is emulated)
    for name, fn in table.items():
        if monkeypatch is not None:
            monkeypatch.setattr(F, name, fn)
        else:
            setattr(F, name, fn)
    CALLS["n"] = 0
    CALLS["gemm_block_n"] = []


# ------------------------------------------------------------------------------------ streams (worst-case reordering)
class LateStream:
    """A side stream that runs everything AS LATE AS THE EVENTS ALLOW: kernels issued under ``torch.cuda.stream(side)`` are
    queued with references to their (live) operand tensors and only executed when another stream waits for an event
    recorded behind them.  A missing wait therefore shows up: the main stream has meanwhile overwritten an operand (or
    reads a result that does not exist yet) and the numbers are wrong."""

    def __init__(self):
        self.queue = []
        self.done = 0            # prefix of the queue that has been executed
        self.reordered = 0       # kernels that ran after later main-stream work had been issued

    def wait_event(self, ev):    # ordering INTO this stream: trivially met, nothing here runs early
        pass

    def run_until(self, pos: int) -> None:
        while self.done < pos:
            fn, issued_at = self.queue[self.done]
            self.done += 1
            if MAIN["issued"] > issued_at:
                self.reordered += 1
            fn()


MAIN = {"issued": 0, "side": None}


class _MainStream:
    def wait_event(self, ev):
        if ev.stream is not None:
            ev.stream.run_until(ev.pos)


class LateEvent:
    def __init__(self, *a, **k):
        self.stream, self.pos = None, 0

    def record(self, stream=None):
        stream = stream if stream is not None else (MAIN["side"] or _MAIN)
        if isinstance(stream, LateStream):
            self.stream, self.pos = stream, len(stream.queue)


_MAIN = _MainStream()


class _StreamCtx:
    def __init__(self, stream):
        self.stream = stream

    def __enter__(self):
        MAIN["side"] = self.stream if isinstance(self.stream, LateStream) else None

    def __exit__(self, *exc):
        MAIN["side"] = None
        return False


def install_late_streams(monkeypatch) -> None:
    """``torch.cuda.{Stream, Event, stream, current_stream}`` replaced by the late-running model above; every emulated
    kernel entry point becomes deferrable (it is queued when issued under a side stream)."""
    from trainingjob_operator_b200.ops import functional as F

    monkeypatch.setattr(torch.cuda, "Stream", LateStream)
    monkeypatch.setattr(torch.cuda, "Event", LateEvent)
    monkeypatch.setattr(torch.cuda, "stream", _StreamCtx)
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a, **k: MAIN["side"] or _MAIN)
    MAIN["issued"], MAIN["side"] = 0, None
    for name in ("gemm", "layernorm_fwd", "layernorm_bwd", "embedding_fwd", "embedding_bwd", "embedding3_fwd",
                 "embedding3_bwd", "softmax_xent", "colsum", "attention_fwd", "attention_bwd", "qkv_gather_colsum", "sumsq",
                 "adamw", "gelu_fwd", "gelu_bwd"):
        real = getattr(F, name)

        def kernel(*a, _real=real, **k):
            side = MAIN["side"]
            if side is not None:
                side.queue.append((lambda: _real(*a, **k), MAIN["issued"]))
                return None
            MAIN["issued"] += 1
            return _real(*a, **k)

        monkeypatch.setattr(F, name, kernel)
