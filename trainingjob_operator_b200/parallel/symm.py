"""Symmetric (peer-mapped + NVSwitch-multicast) gradient buffer for the fused GEMM -> all-reduce path.

The DDP hot op is "weight-gradient GEMM followed by a gradient all-reduce".  Instead of calling a
collective after the GEMM, the gradient buffer is allocated as CUDA symmetric memory with an NVLS
multicast alias (``torch.distributed._symmetric_memory`` provides the allocation/rendezvous plumbing), and
every gradient-producing kernel of the backward pass -- the wgmma wgrad GEMM epilogue, LayerNorm-backward,
the bias column-reduce, the embedding scatter -- issues ``multimem.red.add`` on that alias: the NVSwitch
applies each contribution to all peers' buffers while the math of the next tile proceeds.  When backward
ends, every rank already holds the summed gradient; two device-side barriers per step replace all
gradient collectives.  (The reference has no collective code at all, SURVEY.md §2.5-2.6.)

Falls back (``available == False``) when the platform has no multicast support or the world size is 1.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.distributed as dist


class SymmetricGradBuffer:
    def __init__(self, numel: int, device: torch.device, group=None):
        self.available = False
        self.reason = ""
        self.tensor: Optional[torch.Tensor] = None
        self.handle = None
        self.multicast_ptr = 0
        self._chan = 0
        if not dist.is_initialized() or dist.get_world_size(group) <= 1:
            self.reason = "world size 1"
            return
        try:
            import torch.distributed._symmetric_memory as symm_mem

            pg = group if group is not None else dist.group.WORLD
            try:
                symm_mem.enable_symm_mem_for_group(pg.group_name)
            except Exception:  # noqa: BLE001 - newer torch enables lazily
                pass
            t = symm_mem.empty(numel, dtype=torch.float32, device=device)
            h = symm_mem.rendezvous(t, pg.group_name)
            mc = int(getattr(h, "multicast_ptr", 0) or 0)
            if mc == 0:
                self.reason = "no NVLS multicast support on this platform"
                return
            t.zero_()
            self.tensor, self.handle, self.multicast_ptr = t, h, mc
            self.available = True
        except Exception as e:  # noqa: BLE001
            self.reason = f"{type(e).__name__}: {e}"

    def barrier(self) -> None:
        """Device-side barrier across ranks on the current stream (release/acquire at system scope)."""
        self.handle.barrier(channel=self._chan)
        self._chan = (self._chan + 1) % 2


def shard_bounds(specs, total: int, world: int, align_rows: int = 32, align_flat: int = 256):
    """Ownership bounds of the flat parameter space for ``world`` ranks: ``world + 1`` ascending element offsets, as
    even as the alignment allows.  A bound that falls inside a 2-D tensor is moved to a multiple of ``align_rows`` rows
    of that tensor (the weight-gradient GEMM's epilogue sends 32-row groups to one owner), one inside a 1-D tensor to
    a multiple of ``align_flat`` elements; every bound is a multiple of ``align_flat`` (the AdamW sweep's weight-decay
    mask works in blocks of 256 elements)."""
    bounds = [0]
    for r in range(1, world):
        want = total * r // world
        spec = next((s for s in specs if s.offset <= want < s.offset + s.padded), None)
        if spec is None:
            b = want // align_flat * align_flat
        elif len(spec.shape) == 2:
            unit = align_rows * spec.shape[1]
            while unit % align_flat:
                unit *= 2
            b = spec.offset + min(spec.padded, (want - spec.offset + unit // 2) // unit * unit)
            if b > spec.offset + spec.numel:           # past the last row: hand the whole tensor to the left owner
                b = spec.offset + spec.padded
        else:
            b = spec.offset + (want - spec.offset) // align_flat * align_flat
        bounds.append(max(bounds[-1], min(total, b)))
    bounds.append(total)
    return bounds


class ShardedGradState:
    """Owner-sharded data parallelism over NVLink peer memory (``AITJ_ALLREDUCE=rs``, the default for N > 1).

    The DDP hot op "weight-gradient GEMM, then reduce the gradient" becomes ONE kernel: the flat fp32 gradient buffer
    and the bf16 parameter copy are CUDA symmetric memory (peer-mapped + NVSwitch multicast alias; ``torch``'s
    ``_symmetric_memory`` does the allocation / handle exchange), rank r owns the flat range ``bounds[r]:bounds[r+1]``,
    and

    * every gradient producer -- the wgmma wgrad GEMM epilogue (``EPI_PEER``, split-K partials included), the
      embedding scatter, the pushed 1-D gradients -- ``red.add``s into the OWNER's copy over the peer mapping
      ((N-1)/N of the gradient bytes cross NVLink once; the multicast path delivered N x that);
    * the owner clips (partial square sums are exchanged with one multicast store each) and runs AdamW on its 1/N of
      the fp32 master / moment state only;
    * the refreshed bf16 parameters leave that sweep through the multicast alias -- one store lands in every rank's
      copy -- so the all-gather costs no kernel and no extra pass over memory.

    Three device-side barriers per step (after backward, after the norm exchange, after the optimizer) replace every
    gradient collective; no NCCL kernel runs inside the step, so the whole step is one CUDA graph again and nothing
    competes with the persistent GEMM grids for SMs.  (The reference has no collective code at all, SURVEY.md §2.5-2.6.)
    """

    PARTS = 64       # floats appended to the gradient allocation for the per-rank partial square sums

    def __init__(self, params, device: torch.device, group=None):
        self.available = False
        self.reason = ""
        self.params = params
        if not dist.is_initialized() or dist.get_world_size(group) <= 1:
            self.reason = "world size 1"
            return
        self.world = dist.get_world_size(group)
        self.rank = dist.get_rank(group)
        if self.world > 8:
            self.reason = "more than 8 ranks"
            return
        try:
            import torch.distributed._symmetric_memory as symm_mem

            pg = group if group is not None else dist.group.WORLD
            try:
                symm_mem.enable_symm_mem_for_group(pg.group_name)
            except Exception:  # noqa: BLE001 - newer torch enables lazily
                pass
            total = params.total
            g = symm_mem.empty(total + self.PARTS, dtype=torch.float32, device=device)
            hg = symm_mem.rendezvous(g, pg.group_name)
            w = symm_mem.empty(total, dtype=torch.bfloat16, device=device)
            hw = symm_mem.rendezvous(w, pg.group_name)
            g_mc = int(getattr(hg, "multicast_ptr", 0) or 0)
            w_mc = int(getattr(hw, "multicast_ptr", 0) or 0)
            if g_mc == 0 or w_mc == 0:
                self.reason = "no NVLS multicast support on this platform"
                return
            ptrs = [int(p) for p in hg.buffer_ptrs]
            self.g, self.hg, self.w, self.hw = g, hg, w, hw
            self.g_mc, self.w_mc = g_mc, w_mc
            self.bounds = shard_bounds(params.specs, total, self.world)
            self.lo, self.hi = self.bounds[self.rank], self.bounds[self.rank + 1]
            self.peer_delta = [p - ptrs[self.rank] for p in ptrs]
            g.zero_()
            self._chan = 0
            self._install_tables()
            self.available = True
        except Exception as e:  # noqa: BLE001
            self.reason = f"{type(e).__name__}: {e}"

    def _install_tables(self) -> None:
        import ctypes

        from ..ops import lib

        L = lib.load()
        n = self.world
        delta = (ctypes.c_longlong * 8)(*(self.peer_delta + [0] * (8 - n)))
        bound = (ctypes.c_longlong * 9)(*(self.bounds + [self.bounds[-1]] * (9 - len(self.bounds))))
        for fn in ("aitj_gemm_set_peers", "aitj_fused_set_peers"):
            rc = getattr(L, fn)(ctypes.c_void_p(self.g.data_ptr()), delta, bound, n)
            if rc != 0:
                raise RuntimeError(f"{fn} failed with code {rc}")

    @property
    def parts(self) -> torch.Tensor:
        return self.g[self.params.total:self.params.total + self.world]

    @property
    def parts_mc(self) -> int:
        return self.g_mc + 4 * self.params.total

    def barrier(self) -> None:
        """Device-side barrier across ranks on the current stream (release / acquire at system scope)."""
        self.hg.barrier(channel=self._chan)
        self._chan = (self._chan + 1) % 2
