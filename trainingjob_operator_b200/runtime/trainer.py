"""Training-step driver for the hand-written engines: pinned-host input feed, CUDA-graph replay,
bucketed gradient all-reduce overlapped with backward, fused optimizer sweep, loss read-back.

One ``step()`` is exactly what BASELINE.json's samples/sec counts and what ``bench.py`` times:
H2D copy of this step's tokens from pinned memory -> forward -> backward (+ all-reduce) ->
AdamW -> D2H of the loss.  With a global batch of several micro-batches per rank (``runtime/accumulation.py``),
``accumulate()`` runs forward + backward for every micro-batch but the last, then that step.  The reference operator
has no training loop (SURVEY.md §2.6); this is the launched workers' loop.
"""
from __future__ import annotations

import math
import os
import time
from typing import List, Optional, Tuple

import torch
import torch.distributed as dist

from ..parallel.ddp import BucketAllReducer
from .accumulation import micro_batch_plan


class SyntheticTokens:
    """Synthetic token stream of the named shape, staged in pinned host memory (no dataset access)."""

    def __init__(self, vocab: int, batch: int, seq: int, n_batches: int = 8, seed: int = 0, pin: bool = True):
        g = torch.Generator().manual_seed(seed)
        self.batches = []
        for _ in range(n_batches):
            tok = torch.randint(0, vocab, (batch * seq,), generator=g, dtype=torch.int64)
            tgt = torch.roll(tok, -1)
            if pin and torch.cuda.is_available():
                tok, tgt = tok.pin_memory(), tgt.pin_memory()
            self.batches.append((tok, tgt))
        self.i = 0
        self.bytes_per_step = 2 * batch * seq * 8

    def next(self):
        b = self.batches[self.i % len(self.batches)]
        self.i += 1
        return b


def cosine_lr(step: int, base_lr: float, warmup: int = 10, total: int = 10000, min_ratio: float = 0.1) -> float:
    if step < warmup:
        return base_lr * (step + 1) / warmup
    t = min(1.0, (step - warmup) / max(1, total - warmup))
    return base_lr * (min_ratio + (1 - min_ratio) * 0.5 * (1 + math.cos(math.pi * t)))


class EngineTrainer:
    def __init__(self, engine, lr: float = 3e-4, weight_decay: float = 0.1, max_norm: float = 1.0,
                 use_graph: bool = True, allreduce: Optional[str] = None, group=None, global_batch: int = 0):
        """``global_batch``: samples per optimizer step for the whole job (0: world size x the engine's batch), trained
        in micro-batches of the engine's batch as ``runtime.accumulation.micro_batch_plan`` assigns them."""
        self.engine = engine
        self.lr = lr
        self.weight_decay = weight_decay
        self.max_norm = max_norm
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.group = group
        self.step_count = 0
        self.plan = micro_batch_plan(global_batch, engine.B, self.world, self.rank)
        self.cuda = engine.dev.type == "cuda"
        # rs (default): gradients are reduce-scattered to their owner rank by the kernels that produce them, over NVLink
        # peer memory; sharded AdamW; bf16 parameters all-gathered by multicast stores (parallel/symm.ShardedGradState).
        # mc: every contribution multicast to all ranks (round-1 path).  nccl: bucketed library all-reduce.
        backend = allreduce or os.environ.get("AITJ_ALLREDUCE", "rs")
        self.allreduce_backend = backend if self.world > 1 else "none"
        self.symm = None
        self.shard = None
        self.reducer = None
        if getattr(engine.params, "shard", None) is not None:
            engine.params.detach_shard()      # re-bound after a re-rendezvous: the old group's symmetric buffers go
        if self.world > 1 and backend == "rs" and self.cuda:
            from ..parallel.symm import ShardedGradState

            sh = ShardedGradState(engine.params, engine.dev, group)
            if sh.available:
                engine.params.attach_shard(sh)
                self.shard = sh
                self.allreduce_backend = "rs (wgrad GEMM epilogue red.add to the owner over NVLink peer memory, sharded " \
                                         "AdamW, multicast all-gather of bf16 parameters)"
                sh.barrier()
            else:
                self.allreduce_backend = f"nccl (rs unavailable: {sh.reason})"
                backend = "nccl"
        if self.world > 1 and backend == "mc" and self.cuda and self.plan.accumulates:
            # the multicast path needs every peer at a barrier before each backward: it has no micro-batch step
            raise ValueError("AITJ_ALLREDUCE=mc cannot accumulate micro-batches (global batch "
                             f"{self.plan.global_batch} != {self.world} x {engine.B})")
        if self.world > 1 and backend == "mc" and self.cuda:
            # fused GEMM -> all-reduce: gradients are reduced through the NVSwitch multicast alias by the kernels
            # that produce them (parallel/symm.py); no gradient collective is launched at all
            from ..parallel.symm import SymmetricGradBuffer

            self.symm = SymmetricGradBuffer(engine.params.total, engine.dev, group)
            if self.symm.available:
                engine.params.attach_grad_buffer(self.symm.tensor, self.symm.multicast_ptr)
            else:
                self.allreduce_backend = f"nccl (mc unavailable: {self.symm.reason})"
                self.symm = None
                backend = "nccl"
        if self.world > 1 and self.symm is None and self.shard is None:
            self.reducer = BucketAllReducer(engine.params.g32, engine.grad_buckets(), group, backend)
        engine.grad_hook = self.reducer.hook if self.reducer else None
        if self.reducer is not None:
            reserve = int(os.environ.get("AITJ_DDP_RESERVE_SMS", "0"))
            if reserve > 0:
                from ..ops import functional as F

                engine.bwd_max_ctas = max(2, (F.num_sms() - reserve) // 2 * 2)
                engine.split_k.clear()
        # Without library collectives (1 GPU, or the fused multicast path) the whole step is ONE CUDA graph.  With
        # the NCCL reducer the step is a chain of graphs split where a gradient bucket becomes final; the bucket's
        # all-reduce is launched between two replays on the side stream (capturing NCCL itself deadlocked on
        # the 2-GPU box), so collectives overlap the next segment's math and nothing else is launched eagerly.
        self.use_graph = use_graph and self.cuda
        self.segmented = self.reducer is not None
        # NCCL mode: a bucket's all-reduce starts when its segment's kernels are done, and segments are separate
        # graphs -- each one joins the weight-gradient side stream at its end
        engine.segment_join = self.segmented
        self.seg_graphs = None
        self.graph: Optional[torch.cuda.CUDAGraph] = None
        self.loss_host = torch.zeros(1, dtype=torch.float32)
        if self.cuda:
            self.loss_host = self.loss_host.pin_memory()
        self.graph_error: Optional[str] = None
        self.launches_per_step = 0
        # micro-batch accumulation: the graphs of accumulate() in one-graph mode ("micro", "last" or "idle"), and the
        # sum of this rank's micro-batch losses of the step, kept on the device until the step's one read-back
        self.acc_graphs: Optional[dict] = None
        self.loss_sum = torch.zeros(1, dtype=torch.float32, device=engine.dev)

    # ------------------------------------------------------------------ one step of device work
    def _device_step(self) -> None:
        e = self.engine
        e.forward()
        if self.symm is not None:
            self.symm.barrier()   # every peer finished zeroing its gradients (previous optimizer sweep)
        e.backward()
        if self.symm is not None:
            self.symm.barrier()   # every peer's multimem reductions of this step have landed
        if self.shard is not None:
            self.shard.barrier()  # every contribution to this rank's shard has landed
        if self.reducer:
            self.reducer.wait()
        self._optimizer()
        if self.shard is not None:
            # every rank's bf16 parameters have arrived (next forward) and every shard is zeroed (next backward)
            self.shard.barrier()

    def _optimizer(self) -> None:
        # the gradient buffers hold the sum over the job's k micro-batches of per-micro-batch mean gradients (k = the
        # world size without accumulation)
        self.engine.optimizer_step(lr=self.lr, step=max(1, self.step_count), weight_decay=self.weight_decay,
                                   max_norm=self.max_norm, grad_div=float(self.plan.k), use_dyn=True)

    # ------------------------------------------------------------------ micro-batch accumulation
    def _micro_step(self) -> None:
        """A micro-batch that is not this rank's last of the step: forward + backward only, adding into the gradient
        buffers (no bucket hooks, no collectives, no barriers, no optimizer)."""
        e = self.engine
        e.forward()
        hook, e.grad_hook = e.grad_hook, None
        try:
            e.backward()
        finally:
            e.grad_hook = hook
        self.loss_sum.add_(e.loss)

    def _last_step(self) -> None:
        """This rank's last micro-batch of the step: the single-micro-batch step (gradient sync + optimizer)."""
        self._device_step()
        self.loss_sum.add_(self.engine.loss)

    def _idle_step(self, optimizer=None) -> None:
        """A rank with no micro-batch in this step: the gradient sync and the optimizer of ``_device_step`` on its zero
        gradient, so that it issues the same barriers and bucket all-reduces, in the same order, as the other ranks.
        ``optimizer``: the optimizer's replay when the step runs as graph segments."""
        e = self.engine
        if self.shard is not None:
            self.shard.barrier()
        if self.reducer:
            for buckets, _ in e.backward_segments():
                for b in buckets:
                    self.reducer.hook(b)
            self.reducer.wait()
        (optimizer or self._optimizer)()
        if self.shard is not None:
            self.shard.barrier()

    def _eager_step(self) -> None:
        """One complete optimizer step of this rank's micro-batches, launched eagerly on the current inputs."""
        if self.plan.n == 0:
            self._idle_step()
            return
        for _ in range(self.plan.n - 1):
            self._micro_step()
        self._last_step()

    def _run(self, kind: str) -> None:
        """``kind``: "micro", "last" or "idle" -- from the captured graphs when there are any."""
        if self.seg_graphs is not None:
            if kind == "micro":
                for _, g in self.seg_graphs[:-1]:          # forward and backward segments; no hook, no optimizer
                    g.replay()
                self.loss_sum.add_(self.engine.loss)
            elif kind == "last":
                self._replay_segments()
                self.loss_sum.add_(self.engine.loss)
            else:
                self._idle_step(self.seg_graphs[-1][1].replay)
        elif self.acc_graphs is not None:
            self.acc_graphs[kind].replay()
        else:
            {"micro": self._micro_step, "last": self._last_step, "idle": self._idle_step}[kind]()

    def _warm_up(self) -> None:
        """Two complete steps on a side stream before capture (allocator, cuDNN plans, NCCL channels).  With a fixed
        global batch the state they updated is put back afterwards on every rank -- also at a world size where the step
        is a single micro-batch (k = W): where a job captured its graphs (first step, every rescale) then leaves no mark
        on the optimisation, whatever the world sizes it passes through."""
        P = self.engine.params
        snap = [t.clone() for t in P.state_tensors()] if self.plan.fixed else None
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(2):
                if snap is None:
                    self._device_step()
                else:
                    self._eager_step()
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        if snap is not None:
            # (every rank's state is whole here: the trainer was bound right before the state hand-off.  The last
            # barrier of the warm-up ordered every peer's stores into this rank's bf16 copy before the refresh, and no
            # peer stores into it again before the barrier inside the next optimizer sweep.)
            for t, v in zip(P.state_tensors(), snap):
                t.copy_(v)
            P.refresh_compute_copy()
            self.loss_sum.zero_()
            torch.cuda.synchronize()

    def _capture_accumulating(self) -> None:
        """One-graph mode with accumulation: a graph per kind of micro-batch this rank runs -- "micro" (n >= 2) and
        "last" (n >= 1), or "idle" (n = 0).  Capturing records; it does not execute."""
        from ..ops import lib

        n = self.plan.n
        kinds = {"idle": self._idle_step} if n == 0 else \
            dict(([("micro", self._micro_step)] if n >= 2 else []) + [("last", self._last_step)])
        graphs, launches = {}, {}
        try:
            for kind, fn in kinds.items():
                before = lib.LAUNCHES
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    fn()
                graphs[kind], launches[kind] = g, lib.LAUNCHES - before
            self.acc_graphs = graphs
            self.graph = graphs.get("last") or graphs["idle"]
            self.launches_per_step = launches.get("idle", 0) + launches.get("last", 0) + \
                launches.get("micro", 0) * max(0, n - 1)
        except Exception as ex:  # noqa: BLE001 - fall back to eager launches
            self.acc_graphs = self.graph = None
            self.use_graph = False
            self.graph_error = f"{type(ex).__name__}: {ex}"
            torch.cuda.synchronize()

    def accumulate(self, micro_inputs, read_loss: bool = True) -> Optional[float]:
        """One optimizer step over this rank's ``plan.n`` micro-batches.  ``micro_inputs`` yields each micro-batch's
        inputs in pinned host memory (as ``step`` takes them), and is drawn lazily: the next micro-batch is taken once
        the previous one's copies and work are enqueued, and the iterator runs on after the last one.  Returns the mean
        of this rank's micro-batch losses (NaN when it has none), read back once per step; nothing synchronises with
        the host between micro-batches."""
        e = self.engine
        n = self.plan.n
        self.step_count += 1
        e.set_step_scalars(cosine_lr(self.step_count, self.lr), self.step_count)
        captured = not self.use_graph or self.seg_graphs is not None or self.acc_graphs is not None
        done = 0
        for host in micro_inputs:
            for dst, src in zip(e.input_tensors(), host):
                dst.copy_(src, non_blocking=True)
            if not captured:
                self._capture_segments() if self.segmented else self._capture()
                captured = True
            self._run("micro" if done < n - 1 else "last")
            done += 1
        if done != n:
            raise ValueError(f"rank {self.rank} runs {n} micro-batches per step, {done} were given")
        if n == 0:
            if not captured:
                self._capture_segments() if self.segmented else self._capture()
            self._run("idle")
        if not read_loss:
            return None
        self.loss_host.copy_(self.loss_sum, non_blocking=True)
        self.loss_sum.zero_()
        if self.cuda:
            torch.cuda.current_stream().synchronize()
        return float(self.loss_host[0]) / n if n else float("nan")

    # ------------------------------------------------------------------ graph capture
    def _capture_segments(self) -> None:
        """NCCL mode: [forward] [bwd head] [layer L-1] ... [layer 0] [tail] [optimizer] as separate graphs."""
        from ..ops import lib

        e = self.engine
        self._warm_up()
        saved_hook, e.grad_hook = e.grad_hook, None
        parts = [((), e.forward)] + list(e.backward_segments()) + [(None, self._optimizer)]
        graphs = []
        pool = None
        before = lib.LAUNCHES
        try:
            for buckets, fn in parts:
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g, pool=pool):
                    fn()
                if pool is None:
                    pool = g.pool()
                graphs.append((buckets, g))
            self.seg_graphs = graphs
            self.launches_per_step = lib.LAUNCHES - before
        except Exception as ex:  # noqa: BLE001
            self.seg_graphs = None
            self.use_graph = False
            self.graph_error = f"{type(ex).__name__}: {ex}"
            torch.cuda.synchronize()
        finally:
            e.grad_hook = saved_hook

    def _replay_segments(self) -> None:
        for buckets, g in self.seg_graphs:
            if buckets is None:            # optimizer: every bucket must have been reduced
                self.reducer.wait()
            g.replay()
            for b in buckets or ():
                self.reducer.hook(b)

    def _capture(self) -> None:
        from ..ops import lib

        self._warm_up()
        if self.plan.accumulates:
            self._capture_accumulating()
            return
        before = lib.LAUNCHES
        g = torch.cuda.CUDAGraph()
        try:
            with torch.cuda.graph(g):
                self._device_step()
            self.graph = g
            self.launches_per_step = lib.LAUNCHES - before
        except Exception as ex:  # noqa: BLE001 - fall back to eager replay
            self.graph = None
            self.use_graph = False
            self.graph_error = f"{type(ex).__name__}: {ex}"
            torch.cuda.synchronize()

    def count_launches_eager(self) -> int:
        from ..ops import lib

        before = lib.LAUNCHES
        self._device_step()
        return lib.LAUNCHES - before

    # ------------------------------------------------------------------ public step
    def step(self, *host_inputs: torch.Tensor, read_loss: bool = True) -> Optional[float]:
        """``host_inputs``: this step's inputs in pinned host memory, in the order of ``engine.input_tensors()``
        (GPT-2: tokens, targets; BERT: tokens, token types, MLM labels)."""
        e = self.engine
        self.step_count += 1
        for dst, src in zip(e.input_tensors(), host_inputs):
            dst.copy_(src, non_blocking=True)
        e.set_step_scalars(cosine_lr(self.step_count, self.lr), self.step_count)
        if self.use_graph and self.segmented:
            if self.seg_graphs is None:
                self._capture_segments()
            if self.seg_graphs is not None:
                self._replay_segments()
            else:
                self._device_step()
        elif self.use_graph:
            if self.graph is None:
                self._capture()
                # the two warm-up passes + capture consumed optimizer steps on real data; that is fine for
                # synthetic-data benchmarking and is excluded from timing by the caller's warm-up
            if self.graph is not None:
                self.graph.replay()
            else:
                self._device_step()
        else:
            self._device_step()
        if not read_loss:
            return None
        self.loss_host.copy_(e.loss, non_blocking=True)
        if self.cuda:
            torch.cuda.current_stream().synchronize()
        return float(self.loss_host[0])

    # ------------------------------------------------------------------ evaluation
    def evaluate(self, micro_inputs) -> Tuple[float, int]:
        """Evaluation forwards (``engine.eval_forward``) of this rank's micro-batches, launched eagerly: ``micro_inputs``
        yields each one's inputs in pinned host memory, as ``accumulate`` takes them.  The ranks' (sum of NLL, tokens)
        are summed by one all-reduce on the job's group, which a rank without micro-batches joins too.  Returns the
        job's (sum of NLL, tokens); touches no parameter, gradient or optimizer state."""
        e = self.engine
        e.eval_acc.zero_()
        for host in micro_inputs:
            for dst, src in zip(e.input_tensors(), host):
                dst.copy_(src, non_blocking=True)
            e.eval_forward()
        if self.world > 1:
            dist.all_reduce(e.eval_acc, group=self.group)
        total = e.eval_acc.cpu()
        return float(total[0]), int(total[1])

    def score(self, micro_inputs) -> Tuple[int, int]:
        """Multiple-choice scoring (``engine.score_forward``) of this rank's micro-batches of packed completions,
        launched eagerly: ``micro_inputs`` yields each one's (tokens, targets, doc_start, spans, labels) in pinned host
        memory (``runtime.hellaswag.HellaSwagData.inputs``).  The ranks' (correct, examples) are summed by one all-reduce
        on the job's group, which a rank without micro-batches joins too.  Touches no parameter, gradient or optimizer
        state."""
        e = self.engine
        e.choice_acc.zero_()
        for tok, tgt, doc_start, spans, labels in micro_inputs:
            e.tok.copy_(tok, non_blocking=True)
            e.tgt.copy_(tgt, non_blocking=True)
            e.score_forward(doc_start, spans.to(e.dev, non_blocking=True), labels.to(e.dev, non_blocking=True),
                            spans.shape[0])
        if self.world > 1:
            dist.all_reduce(e.choice_acc, group=self.group)
        total = e.choice_acc.cpu()
        return int(total[0]), int(total[1])

    def state_tensors(self) -> List[torch.Tensor]:
        return self.engine.params.state_tensors()
