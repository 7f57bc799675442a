"""Flat parameter / gradient / optimizer-state storage for the hand-written training engines.

Everything a worker trains lives in five contiguous device buffers laid out for 80 GB of HBM3 and
one-sweep kernels: fp32 master weights ``p32``, their bf16 compute copy ``p16`` (what the wgmma
GEMMs read through TMA), fp32 gradients ``g32`` (wgrad GEMMs ``red.add`` into it, split-K and
micro-batches accumulate for free), and AdamW moments ``m`` / ``v``.  Tensors are padded to 256
elements so the per-256-element weight-decay mask of the AdamW kernel lines up, and the contiguous
layout makes gradient buckets plain slices (DDP all-reduce without a flatten/unflatten copy).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, Iterable, List, Tuple

import torch

ALIGN = 256


@dataclass
class ParamSpec:
    name: str
    shape: Tuple[int, ...]
    decay: bool
    init: str = "normal"      # normal | zeros | ones
    std: float = 0.02
    offset: int = 0
    numel: int = 0
    padded: int = 0


class FlatParams:
    def __init__(self, specs: Iterable[ParamSpec], device, with_optimizer_state: bool = True, seed: int = 0):
        self.specs: List[ParamSpec] = list(specs)
        off = 0
        for s in self.specs:
            n = 1
            for d in s.shape:
                n *= d
            s.numel = n
            s.padded = (n + ALIGN - 1) // ALIGN * ALIGN
            s.offset = off
            off += s.padded
        self.total = off
        self.device = torch.device(device)
        self.p32 = torch.zeros(self.total, dtype=torch.float32, device=self.device)
        self.p16 = torch.zeros(self.total, dtype=torch.bfloat16, device=self.device)
        self.g32 = torch.zeros(self.total, dtype=torch.float32, device=self.device)
        if with_optimizer_state:
            self.m = torch.zeros(self.total, dtype=torch.float32, device=self.device)
            self.v = torch.zeros(self.total, dtype=torch.float32, device=self.device)
        else:
            self.m = self.v = None
        mask = torch.zeros(self.total // ALIGN, dtype=torch.uint8)
        for s in self.specs:
            if s.decay:
                mask[s.offset // ALIGN:(s.offset + s.padded) // ALIGN] = 1
        self.wd_mask = mask.to(self.device)
        self.by_name: Dict[str, ParamSpec] = {s.name: s for s in self.specs}
        self.mc_base = 0
        self.small_range = None
        self.g_small = None
        self.shard = None          # parallel.symm.ShardedGradState when gradients are owner-sharded over NVLink
        self.init_parameters(seed)

    def init_parameters(self, seed: int = 0) -> None:
        """Random-init in place with a generator ON THE DEVICE OF THE BUFFERS.  Drawing GPT-2 small's 124 M normals from a
        CPU generator and copying them tensor by tensor took 2.5 s of a single core per worker (more than half of a
        warm-started worker's time to its first step); the device generator fills the flat buffer in milliseconds.  Every
        rank uses the same seed (Philox: same values on every GPU), and the elected state hand-off follows anyway."""
        import os

        on_host = os.environ.get("AITJ_PARAM_INIT") == "cpu"     # the numerics self-check keeps its historical weights
        gen = torch.Generator(device="cpu" if on_host else self.p32.device)    # the buffer's concrete device (cuda:N)
        gen.manual_seed(seed)
        for s in self.specs:
            view = self.p32[s.offset:s.offset + s.numel].view(s.shape)
            if s.init == "zeros":
                view.zero_()
            elif s.init == "ones":
                view.fill_(1.0)
            elif on_host:
                view.copy_(torch.randn(s.shape, generator=gen, dtype=torch.float32) * s.std)
            else:
                view.normal_(0.0, s.std, generator=gen)
        self.refresh_compute_copy()

    def refresh_compute_copy(self) -> None:
        self.p16.copy_(self.p32)

    # -- views ---------------------------------------------------------------------------------
    def _view(self, buf: torch.Tensor, name: str) -> torch.Tensor:
        s = self.by_name[name]
        return buf[s.offset:s.offset + s.numel].view(s.shape)

    def w16(self, name: str) -> torch.Tensor:
        return self._view(self.p16, name)

    def w32(self, name: str) -> torch.Tensor:
        return self._view(self.p32, name)

    def grad(self, name: str):
        """Where gradient-producing kernels accumulate ``name``'s gradient: the local fp32 slice, or -- when a
        symmetric buffer with an NVSwitch multicast alias is attached -- that alias (reduce-to-all-peers)."""
        if self.shard is not None:
            s = self.by_name[name]
            if len(s.shape) == 1 and self.small_range is not None:
                a = s.offset - self.small_range[0]
                return self.g_small[a:a + s.numel]
            from ..ops.functional import PeerView

            return PeerView(self._view(self.g32, name))
        if self.mc_base:
            from ..ops.functional import RawView

            s = self.by_name[name]
            if len(s.shape) == 1 and self.small_range is not None:
                # small 1-D params are accumulated locally (scalar atomics) and pushed once per step
                a = s.offset - self.small_range[0]
                return self.g_small[a:a + s.numel]
            return RawView(self.mc_base + 4 * s.offset, s.shape, torch.float32)
        return self._view(self.g32, name)

    def local_grad(self, name: str) -> torch.Tensor:
        return self._view(self.g32, name)

    def attach_grad_buffer(self, buf: torch.Tensor, multicast_ptr: int = 0) -> None:
        """Replace the gradient buffer (e.g. by a symmetric-memory allocation) and set its multicast alias."""
        assert buf.numel() >= self.total and buf.dtype == torch.float32
        self.g32 = buf[: self.total]
        self.g32.zero_()
        self.mc_base = int(multicast_ptr or 0)
        self.small_range = None
        if self.mc_base:
            one_d = [s for s in self.specs if len(s.shape) == 1]
            if one_d:
                lo = min(s.offset for s in one_d)
                hi = max(s.offset + s.padded for s in one_d)
                # only valid when the 1-D parameters form one contiguous tail region of the layout
                if all(len(s.shape) == 1 for s in self.specs if lo <= s.offset < hi):
                    self.small_range = (lo, hi)
                    self.g_small = torch.zeros(hi - lo, dtype=torch.float32, device=self.device)

    def _small_region(self) -> None:
        """1-D parameters (biases, LayerNorm) are accumulated locally with scalar atomics and sent once per step; only
        possible when they form one contiguous tail region of the layout."""
        self.small_range = None
        one_d = [s for s in self.specs if len(s.shape) == 1]
        if one_d:
            lo = min(s.offset for s in one_d)
            hi = max(s.offset + s.padded for s in one_d)
            if all(len(s.shape) == 1 for s in self.specs if lo <= s.offset < hi):
                self.small_range = (lo, hi)
                self.g_small = torch.zeros(hi - lo, dtype=torch.float32, device=self.device)

    def attach_shard(self, shard) -> None:
        """Owner-sharded mode: gradients and the bf16 parameter copy move into ``shard``'s symmetric buffers."""
        self.g32 = shard.g[: self.total]
        self.g32.zero_()
        shard.w.copy_(self.p16)
        self.p16 = shard.w
        self.mc_base = 0
        self.shard = shard
        self._small_region()
        if self.small_range is None:
            raise RuntimeError("owner-sharded gradients need the 1-D parameters in one tail region of the layout")

    def detach_shard(self) -> None:
        """Back to private buffers (the world shrank to one rank, or another gradient path was selected)."""
        if self.shard is None:
            return
        p16 = torch.empty(self.total, dtype=torch.bfloat16, device=self.device)
        p16.copy_(self.p16)
        self.p16 = p16
        self.g32 = torch.zeros(self.total, dtype=torch.float32, device=self.device)
        self.shard = None
        self.small_range = None
        self.g_small = None

    def push_small_grads(self) -> None:
        """Multicast mode: send the locally accumulated 1-D parameter gradients to every peer (one kernel); owner-sharded
        mode: to the ranks that own them."""
        if self.shard is not None:
            from ..ops import functional as F

            lo, hi = self.small_range
            F.peer_push(self.g32[lo:hi], self.g_small)
            return
        if self.mc_base and self.small_range is not None:
            from ..ops import functional as F

            lo, hi = self.small_range
            F.mc_push(self.mc_base + 4 * lo, self.g_small, hi - lo)

    def range_of(self, first: str, last: str) -> Tuple[int, int]:
        a, b = self.by_name[first], self.by_name[last]
        return a.offset, b.offset + b.padded

    def num_parameters(self) -> int:
        return sum(s.numel for s in self.specs)

    # -- state (checkpoint / elastic hand-off) ------------------------------------------------------
    def state_tensors(self) -> List[torch.Tensor]:
        out = [self.p32]
        if self.m is not None:
            out += [self.m, self.v]
        return out

    def state_dict(self) -> Dict[str, torch.Tensor]:
        d = {"p32": self.p32}
        if self.m is not None:
            d["m"] = self.m
            d["v"] = self.v
        return d

    def load_state_dict(self, d: Dict[str, torch.Tensor]) -> None:
        self.p32.copy_(d["p32"])
        if self.m is not None and "m" in d:
            self.m.copy_(d["m"])
            self.v.copy_(d["v"])
        self.refresh_compute_copy()
