"""Which micro-batches a rank trains in one optimizer step, for a fixed global batch at any world size.

A job trains ``G`` samples per optimizer step (``--global-batch``), in ``k = G / B`` micro-batches of the per-GPU batch
``B``.  At world size ``W``, rank ``r`` runs micro-batches ``j = r, r + W, r + 2W, ... < k``, so ranks differ by at most
one micro-batch and a rank with ``r >= k`` runs none.  Micro-batch ``j`` of the step at sample position ``pos`` reads
samples ``[pos + j*B, pos + (j+1)*B)``, and the step advances the position by ``G``.  Every gradient is summed over the
job's micro-batches and divided by ``k``, so the update depends on ``G`` and the sample sequence, not on ``W``.

With ``G = W*B`` every rank runs exactly micro-batch ``r``: rank ``r`` reads ``[pos + r*B, pos + (r+1)*B)``, the
gradient is divided by ``W``, and the trainers take their single-micro-batch step.  That is also the default
(``global_batch=0``); a plan whose global batch was given is ``fixed``, which it stays when a rescale makes ``k = W``.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Tuple


@dataclass(frozen=True)
class MicroBatchPlan:
    global_batch: int      # G: samples per optimizer step, whole job
    batch: int             # B: samples per micro-batch
    world: int             # W
    rank: int              # r
    micro: Tuple[int, ...]  # the micro-batch indices j this rank runs, ascending
    fixed: bool = False    # the global batch was given (``--global-batch``), not derived from the world size

    @property
    def k(self) -> int:
        """Micro-batches per optimizer step, whole job; the optimizer divides the summed gradient by it."""
        return self.global_batch // self.batch

    @property
    def n(self) -> int:
        """Micro-batches this rank runs per optimizer step (``ceil(k/W)`` or ``floor(k/W)``; 0 when ``rank >= k``)."""
        return len(self.micro)

    @property
    def accumulates(self) -> bool:
        """False exactly when every rank runs one micro-batch (``G = W*B``): the trainers' single-micro-batch step."""
        return self.k != self.world

    def first_sample(self, position: int, j: int) -> int:
        """First sample of micro-batch ``j`` of the step at sample position ``position``."""
        return position + j * self.batch

    def windows(self, position: int):
        """[(first sample, count)] this rank reads in the step at ``position``, in the order it trains them."""
        return [(self.first_sample(position, j), self.batch) for j in self.micro]


def micro_batch_plan(global_batch: int, batch: int, world: int, rank: int) -> MicroBatchPlan:
    """The plan of rank ``rank`` of ``world`` for ``global_batch`` samples per step in micro-batches of ``batch``
    (``global_batch=0``: ``world * batch``)."""
    if batch < 1 or world < 1 or not 0 <= rank < world:
        raise ValueError(f"bad micro-batch plan arguments: batch {batch}, world {world}, rank {rank}")
    G = global_batch or world * batch
    if G % batch:
        raise ValueError(f"the global batch {G} is not a multiple of the per-GPU batch {batch}")
    k = G // batch
    return MicroBatchPlan(G, batch, world, rank, tuple(range(rank, k, world)), fixed=bool(global_batch))
