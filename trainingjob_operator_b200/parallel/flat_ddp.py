"""DDP for ordinary ``nn.Module`` models (MNIST CNN, ResNet-50) on the same flat-buffer machinery.

Parameters are re-pointed at views of one flat fp32 buffer and ``.grad`` at views of one flat
gradient buffer, so (a) gradient buckets are slices reduced as soon as autograd finishes them
(post-accumulate hooks -> ``BucketAllReducer``), (b) the optimizer is the single-sweep fused AdamW /
SGD kernel over the whole model, (c) elastic state hand-off is three broadcasts.  This is the
launched-worker side of the reference's "N identical trainer replicas" wiring (pod.go:553-628); the
reference itself has no data-parallel code (SURVEY.md §2.4).
"""
from __future__ import annotations

from typing import Dict, List, Tuple

import torch
import torch.distributed as dist

from .ddp import BucketAllReducer

ALIGN = 256


class FlatDDP:
    def __init__(self, module: torch.nn.Module, bucket_bytes: int = 25 << 20, group=None, backend: str = "nccl",
                 weight_decay: float = 0.0, lr: float = 1e-3, optimizer: str = "adamw", momentum: float = 0.9,
                 overlap: bool = True):
        """``overlap=False``: no per-bucket hooks -- the caller replays forward + backward as one CUDA graph (Python
        hooks do not run on a replay) and ``finish_backward`` reduces the whole flat gradient buffer with one collective."""
        self.module = module
        self.overlap = overlap
        self.group = group
        self.lr, self.weight_decay, self.momentum = lr, weight_decay, momentum
        self.optimizer = optimizer
        params = [p for p in module.parameters() if p.requires_grad]
        dev = params[0].device
        self.dev = dev
        offs, off = [], 0
        for p in params:
            offs.append(off)
            off += (p.numel() + ALIGN - 1) // ALIGN * ALIGN
        self.total = off
        self.p32 = torch.zeros(off, dtype=torch.float32, device=dev)
        self.g32 = torch.zeros(off, dtype=torch.float32, device=dev)
        self.m = torch.zeros(off, dtype=torch.float32, device=dev)
        self.v = torch.zeros(off, dtype=torch.float32, device=dev) if optimizer == "adamw" else None
        self.p16 = torch.zeros(off, dtype=torch.bfloat16, device=dev) if dev.type == "cuda" else None
        mask = torch.zeros(off // ALIGN, dtype=torch.uint8)
        self.params = params
        for p, o in zip(params, offs):
            n = p.numel()
            self.p32[o:o + n].copy_(p.detach().reshape(-1).float())
            p.data = self.p32[o:o + n].view(p.shape)
            p.grad = self.g32[o:o + n].view(p.shape)
            if p.dim() > 1:
                mask[o // ALIGN:(o + n + ALIGN - 1) // ALIGN] = 1
        self.wd_mask = mask.to(dev)
        # buckets in reverse registration order (~ the order autograd produces gradients)
        buckets: List[Tuple[str, int, int]] = []
        self._bucket_of: Dict[int, int] = {}
        self._pending: List[int] = []
        end = off
        cur_start, count, bi = off, 0, 0
        for idx in range(len(params) - 1, -1, -1):
            cur_start = offs[idx]
            self._bucket_of[idx] = bi
            count += 1
            if (end - cur_start) * 4 >= bucket_bytes or idx == 0:
                buckets.append((f"b{bi}", cur_start, end))
                self._pending.append(count)
                end, count, bi = cur_start, 0, bi + 1
        self.buckets = buckets
        self._todo = list(self._pending)
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.reducer = BucketAllReducer(self.g32, buckets, group, backend, min_bucket_bytes=0) \
            if self.world > 1 else None
        self._hooked = False
        # micro-batch accumulation: ``k`` micro-batches per optimizer step, whole job (None: one per rank, k = world);
        # ``sync`` is cleared while a rank runs a micro-batch that is not its last of the step, so that the bucket hooks
        # leave the partial sums alone
        self.k = None
        self.sync = True
        if self.reducer is not None and overlap:
            for idx, p in enumerate(params):
                p.register_post_accumulate_grad_hook(self._make_hook(idx))
            self._hooked = True
        self.step_count = 0

    def _make_hook(self, idx: int):
        b = self._bucket_of[idx]

        def hook(_p):
            if self.reducer is None or not self.sync:
                return
            self._todo[b] -= 1
            if self._todo[b] == 0:
                self.reducer.hook(f"b{b}")

        return hook

    def finish_backward(self) -> None:
        if self.reducer is not None and not self.overlap:
            self.reducer.all_reduce_all()
            return
        if self.reducer is not None:
            # buckets whose parameters received no gradient this step still have to be reduced
            for b, left in enumerate(self._todo):
                if left > 0:
                    self.reducer.hook(f"b{b}")
            self.reducer.wait()
            self._todo = list(self._pending)

    def discard_step(self) -> None:
        """Forget a step that died in its gradient all-reduce (a peer was lost): the flat gradient buffer holds local or
        partly reduced sums that must not leak into the next step; parameters and moments were not touched yet."""
        if self.reducer is not None:
            self.reducer._works.clear()
        self._todo = list(self._pending)
        self.g32.zero_()

    def step(self) -> None:
        """Fused optimizer sweep (+ gradient zeroing); the summed gradients are divided by the number of micro-batches of
        the step, whole job (the world size without accumulation): a mean of per-micro-batch mean gradients."""
        self.step_count += 1
        div = float(self.k or self.world)
        if self.dev.type == "cuda" and self.optimizer == "adamw":
            from ..ops import functional as F

            F.adamw(self.p32, self.g32, self.m, self.v, self.p16, self.wd_mask, lr=self.lr, beta1=0.9, beta2=0.999,
                    eps=1e-8, weight_decay=self.weight_decay, step=self.step_count, grad_div=div,
                    zero_grad=True)
            return
        with torch.no_grad():
            g = self.g32 / div
            if self.optimizer == "adamw":
                b1, b2 = 0.9, 0.999
                self.m.mul_(b1).add_(g, alpha=1 - b1)
                self.v.mul_(b2).addcmul_(g, g, value=1 - b2)
                mh = self.m / (1 - b1 ** self.step_count)
                vh = self.v / (1 - b2 ** self.step_count)
                self.p32.add_(mh / (vh.sqrt() + 1e-8), alpha=-self.lr)
            else:
                self.m.mul_(self.momentum).add_(g)
                self.p32.add_(self.m, alpha=-self.lr)
            self.g32.zero_()

    def state_tensors(self) -> List[torch.Tensor]:
        return [t for t in (self.p32, self.m, self.v) if t is not None]
