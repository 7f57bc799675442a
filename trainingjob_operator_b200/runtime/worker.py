"""Worker runtime: the process the node agent launches for every replica of a benchmark job.

Reads the environment contract injected by the controller (the reference's 13 variables,
/root/reference/pkg/controller/pod.go:548-652, plus the torch / elastic dialect added in
``controller/pod.py``), joins ``torch.distributed`` (NCCL over NVLink 5 / NVSwitch on GPUs, gloo on
CPU), builds the requested model and runs the measured training loop:

* every step: H2D of the step's inputs from pinned memory, forward, backward + bucketed all-reduce,
  fused optimizer sweep, D2H of the loss;
* timing: W untimed warm-up steps, then exactly K steps bracketed by barrier + synchronize, CUDA
  events on the device, max over ranks; rank 0 writes the result JSON and patches it onto the job;
* elastic (``runtime.elastic``): a side thread watches ``status.rendezvous``; at a step boundary all
  ranks agree on the newest generation, tear the process group down and re-rendezvous with the new
  world size; survivors keep params / optimizer state / step on the device and broadcast them to
  joiners; ranks that fall out of range leave with exit 0;
* restart: ``TRAININGJOB_REPLICA_RESTARTCOUNT`` > 0 => resume from the newest checkpoint written (asynchronously,
  ``runtime.checkpoint``) by rank 0 every ``--ckpt-every`` steps (SURVEY.md §5.4);
* ``faultTolerant`` elastic jobs: a collective that fails because a peer died does not end the process -- the step is
  discarded, the group dropped, and the loop continues on the controller's next generation (``runtime.rendezvous``).
"""
from __future__ import annotations

import argparse
import gc
import json
import os
import signal
import sys
import time
from typing import Any, Dict, List, Optional

import torch
import torch.distributed as dist

from ..models.gpt2 import GPT2_MODELS
from ..ops import lib as oplib
from .elastic import ElasticWatcher, env_int, rendezvous_from_env
from .rendezvous import (StaleGeneration, StallBreaker, guarded, heartbeat, init_process_group,  # noqa: F401
                         max_over_ranks, rendezvous, sync_state, teardown_group, wait_for_newer_generation)
from .trainer import EngineTrainer, SyntheticTokens


# ------------------------------------------------------------------------------------ adapters
class EngineAdapter:
    """GPT-2 / BERT-shaped transformer on the hand-written engine (CUDA only)."""

    def __init__(self, name: str, batch: int, seq: int, args, device: str = "cuda"):
        """``device``: always "cuda" in a worker (``build_adapter``); the CPU dry-run tests pass "cpu" together with
        emulated kernel entry points (tests/kernel_emulation.py) to execute the adapter's control flow."""
        from ..models.gpt2 import GPT2Engine, flops_per_token, gpt2_config

        if name in ("bert", "bert-tiny"):
            # the real thing: word + position + token-type embeddings, post-LN bidirectional encoder, MLM head and loss
            from ..models.bert import BertConfig, BertEngine, SyntheticMLM, bert_flops_per_token

            cfg = BertConfig.base() if name == "bert" else BertConfig.tiny()
            seq = min(seq, cfg.block_size)
            self.engine = BertEngine(cfg, batch, seq, device, seed=args.seed, gemm_backend=args.gemm)
            self.data = SyntheticMLM(cfg.vocab_size, batch, seq, n_batches=4, seed=args.seed + 1, pin=device != "cpu")
            self.flops_per_step = bert_flops_per_token(cfg, seq) * batch * seq
        else:
            if name not in GPT2_MODELS:
                raise ValueError(name)
            cfg = gpt2_config(name)
            seq = min(seq, cfg.block_size)
            doc_mask = bool(getattr(args, "doc_mask", False))
            self.engine = GPT2Engine(cfg, batch, seq, device, seed=args.seed, gemm_backend=args.gemm, causal=True,
                                     doc_mask=doc_mask)
            if getattr(args, "data", ""):
                from .data import TokenFileData

                # samples consumed by the whole job; rank r of W reads [pos + r*B, pos + (r+1)*B) at a step
                self.data_position = 0
                self.data = TokenFileData(args.data, seq, cfg.vocab_size, doc_mask=doc_mask, eot=args.eot_token,
                                          pin=device != "cpu")
            else:
                self.data = SyntheticTokens(cfg.vocab_size, batch, seq, n_batches=4, seed=args.seed + 1)
            self.flops_per_step = flops_per_token(cfg, seq) * batch * seq
            if getattr(args, "eval_data", ""):
                from .data import DataError, TokenFileData

                # held-out windows [0, eval_samples) of their own stream: no position, so nothing to hand off or save
                self.eval_data = TokenFileData(args.eval_data, seq, cfg.vocab_size, doc_mask=doc_mask,
                                               eot=args.eot_token, pin=device != "cpu")
                self.eval_samples = args.eval_samples or 20 * batch
                if self.eval_samples > self.eval_data.n_windows:
                    raise DataError(f"--eval-samples {self.eval_samples}: --eval-data {args.eval_data!r} holds only "
                                    f"{self.eval_data.n_windows} windows of {seq + 1} tokens")
            if getattr(args, "hellaswag", ""):
                from .hellaswag import HellaSwagData

                # multiple-choice scoring: the file's completions packed into micro-batches once, pinned
                self.hellaswag = HellaSwagData(args.hellaswag, cfg.vocab_size, batch, seq, pin=device != "cpu")
            if getattr(args, "generate_every", None) is not None:
                # text generation at step boundaries: a generator of its own (buffers, KV caches) on the engine's
                # weights, built at the first generation
                self.generator = None
                self.tokenizer = None
                if args.tokenizer:
                    from .tokenizer import Tokenizer, TokenizerError

                    self.tokenizer = Tokenizer(args.tokenizer)
                    if self.tokenizer.vocab_size < cfg.vocab_size:
                        raise TokenizerError(f"{args.tokenizer}: {self.tokenizer.vocab_size} tokens, fewer than the "
                                             f"{cfg.vocab_size} of {cfg.name}")
        self.cfg = cfg
        self.batch, self.seq = batch, seq
        self.h2d_bytes = self.data.bytes_per_sample * batch if hasattr(self, "data_position") else \
            self.data.bytes_per_step
        self.d2h_bytes = 4
        self.trainer: Optional[EngineTrainer] = None
        self.args = args
        self.describe = {"model": cfg.name, "seq_len": seq, "params": self.engine.num_parameters(),
                         "gemm": args.gemm}
        if hasattr(self, "data_position"):
            self.describe.update(data=args.data, doc_mask=self.engine.doc_mask, windows=self.data.n_windows)
        if hasattr(self, "eval_data"):
            self.describe.update(eval_data=args.eval_data, eval_samples=self.eval_samples)
        if hasattr(self, "hellaswag"):
            self.describe.update(hellaswag=args.hellaswag, hellaswag_examples=self.hellaswag.examples,
                                 hellaswag_micro_batches=self.hellaswag.micro_batches)

    def bind(self, group=None, warm_up: bool = False) -> None:
        """(Re-)build the trainer for the current process group; the micro-batch plan follows its world size.
        ``warm_up``: a joiner's throw-away steps before it enters the job, one micro-batch each."""
        old = self.trainer
        # a faultTolerant job survives the loss of a peer in place, which needs every rank to hold the whole optimizer
        # state and a collective that can be aborted: library all-reduce instead of the owner-sharded peer-memory path
        allreduce = "nccl" if os.environ.get("AITJ_FAULT_TOLERANT") == "1" and "AITJ_ALLREDUCE" not in os.environ else None
        self.trainer = EngineTrainer(self.engine, lr=self.args.lr, use_graph=not self.args.no_graph, group=group,
                                     allreduce=allreduce,
                                     global_batch=0 if warm_up else getattr(self.args, "global_batch", 0))
        if old is not None:
            self.trainer.step_count = old.step_count

    @property
    def plan(self):
        return self.trainer.plan

    def train_step(self) -> float:
        plan = getattr(self.trainer, "plan", None)
        if plan is not None and plan.accumulates:
            return self.trainer.accumulate(self._micro_inputs())
        if not hasattr(self, "data_position"):
            return self.trainer.step(*self.data.next())
        world, rank = self.trainer.world, self.trainer.rank
        host = self.data.stage(self.data_position + rank * self.batch, self.batch)
        loss = self.trainer.step(*host)
        self.data.in_flight()
        self.data_position += world * self.batch     # not reached when the step fails: a discarded step reads again
        return loss

    def _micro_inputs(self):
        """This rank's micro-batches of the step, staged one at a time as the trainer takes them; the data position moves
        by the global batch once the last one is enqueued.  Without ``--data`` each takes the next synthetic batch."""
        plan = self.trainer.plan
        if not hasattr(self, "data_position"):
            for _ in range(plan.n):
                yield self.data.next()
                heartbeat()
            return
        read = []
        for first, count in plan.windows(self.data_position):
            yield self.data.stage(first, count)
            self.data.in_flight()
            read += self.data.samples_read
            heartbeat()                    # a long accumulated step must not look like a hang to the agent
        self.samples_read = read
        self.data_position += plan.global_batch

    def eval_plan(self):
        """This rank's share of the evaluation: the held-out windows [0, S) cut into ceil(S / B) micro-batches, assigned
        to the ranks as ``runtime.accumulation`` assigns a step's micro-batches."""
        from .accumulation import micro_batch_plan

        B = self.batch
        k = -(-self.eval_samples // B)
        return micro_batch_plan(k * B, B, self.trainer.world, self.trainer.rank)

    def _eval_inputs(self, progress=None):
        S = self.eval_samples
        for first, count in self.eval_plan().windows(0):
            yield self.eval_data.stage(first, count, min(count, S - first))   # past S: token 0, target -1
            self.eval_data.in_flight()
            heartbeat()
            if progress is not None:
                progress()

    def evaluate(self, progress=None) -> Dict[str, Any]:
        """The job's mean NLL per token over the held-out windows (collective: every rank calls it).  ``progress`` is
        called after each of this rank's micro-batches is enqueued."""
        total, tokens = self.trainer.evaluate(self._eval_inputs(progress))
        return {"loss": total / max(1, tokens), "tokens": tokens, "samples": self.eval_samples}

    def score(self, progress=None) -> Dict[str, Any]:
        """The job's HellaSwag accuracy (collective: every rank calls it).  ``progress`` is called after each of this
        rank's micro-batches is enqueued."""
        hs = self.hellaswag

        def inputs():
            for k in hs.plan(self.trainer.world, self.trainer.rank):
                yield hs.inputs(k)
                heartbeat()
                if progress is not None:
                    progress()

        correct, examples = self.trainer.score(inputs())
        return {"correct": correct, "examples": examples, "acc": correct / max(1, examples)}

    def generate(self, step: int, progress=None) -> Dict[str, Any]:
        """``--generate-count`` sequences of the prompt and ``--generate-tokens`` new tokens, sampled with the seed of this
        step (``generation_seed``).  Local: every rank computes the same from its own copy of the weights.  ``progress``
        is called every few tokens."""
        from ..models.generate import GPT2Generator, generation_seed

        a = self.args
        if self.generator is None:
            self.generator = GPT2Generator(self.engine, a.generate_count, len(a.generate_prompt) + a.generate_tokens)
        seed = generation_seed(a.seed, step)

        def tick(_tokens):
            heartbeat()
            if progress is not None:
                progress()

        toks = self.generator.generate(a.generate_prompt, a.generate_tokens, temperature=a.temperature, top_k=a.top_k,
                                       seed=seed, use_graph=not a.no_graph and self.engine.dev.type == "cuda",
                                       progress=tick)
        rec: Dict[str, Any] = {"seed": seed, "tokens": toks.tolist()}
        if self.tokenizer is not None:
            rec["text"] = [self.tokenizer.decode(t) for t in rec["tokens"]]
        return rec

    def discard_step(self) -> None:
        self.engine.params.g32.zero_()
        if self.engine.params.g_small is not None:
            self.engine.params.g_small.zero_()
        if self.trainer is not None:
            self.trainer.loss_sum.zero_()

    def prepare_state(self) -> None:
        """Collective.  With the owner-sharded optimizer every rank only keeps its own range of the fp32 master weights
        and moments current: gather them so that ``state_tensors`` is the whole state on every rank (before a
        checkpoint, before the process group is re-formed)."""
        sh = self.engine.params.shard
        if sh is None or not dist.is_initialized():
            return
        P = self.engine.params
        for r in range(sh.world):
            a, b = sh.bounds[r], sh.bounds[r + 1]
            if b > a:
                for t in (P.p32, P.m, P.v):
                    dist.broadcast(t[a:b], src=r)

    def state_tensors(self) -> List[torch.Tensor]:
        return self.engine.params.state_tensors()

    def after_state_load(self) -> None:
        self.engine.params.refresh_compute_copy()

    @property
    def step_count(self) -> int:
        return self.trainer.step_count if self.trainer else 0

    @step_count.setter
    def step_count(self, v: int) -> None:
        if self.trainer:
            self.trainer.step_count = v

    def launches_per_step(self) -> int:
        return self.trainer.launches_per_step or 0

    @property
    def gradient_sync(self) -> str:
        return self.trainer.allreduce_backend

    def graph_report(self, world: int) -> Dict[str, Any]:
        """The result's CUDA-graph and all-reduce fields."""
        t = self.trainer
        return {"cuda_graph": bool(t.graph or t.seg_graphs), "graph_segments": len(t.seg_graphs or []) or None,
                "graph_error": t.graph_error, "allreduce": t.allreduce_backend}


class TorchAdapter:
    """nn.Module models (MNIST CNN, ResNet-50, CPU MLP) through ``parallel.flat_ddp``."""

    def __init__(self, name: str, batch: int, args, device: torch.device):
        from ..models.mnist_cnn import MLP, MnistCNN

        self.name, self.batch, self.dev, self.args = name, batch, device, args
        g = torch.Generator().manual_seed(args.seed + 1)
        if name == "mnist":
            self.module = MnistCNN()
            shape, ncls = (1, 28, 28), 10
        elif name == "resnet50":
            from ..models.resnet50 import build_resnet50

            self.module = build_resnet50()
            shape, ncls = (3, 224, 224), 1000
        elif name == "mlp":
            self.module = MLP()
            shape, ncls = (64,), 10
        else:
            raise ValueError(name)
        torch.manual_seed(args.seed)
        self.module = self.module.to(device)
        self.channels_last = device.type == "cuda" and len(shape) == 3
        if self.channels_last:
            self.module = self.module.to(memory_format=torch.channels_last)
        pin = device.type == "cuda"
        self.batches = []
        for _ in range(4):
            x = torch.randn(batch, *shape, generator=g)
            y = torch.randint(0, ncls, (batch,), generator=g)
            if pin:
                x, y = x.pin_memory(), y.pin_memory()
            self.batches.append((x, y))
        self.i = 0
        self.x_dev = torch.empty(batch, *shape, device=device)
        if self.channels_last:
            self.x_dev = self.x_dev.contiguous(memory_format=torch.channels_last)
        self.y_dev = torch.empty(batch, dtype=torch.int64, device=device)
        self.h2d_bytes = self.batches[0][0].numel() * 4 + batch * 8
        self.d2h_bytes = 4
        self.ddp = None
        self._steps = 0
        self.loss_host = torch.zeros(1).pin_memory() if pin else torch.zeros(1)
        self.describe = {"model": name, "params": sum(p.numel() for p in self.module.parameters())}
        self.flops_per_step = 0.0
        self.use_graph, self.graph, self.graph_error = False, None, None

    def bind(self, group=None, warm_up: bool = False) -> None:
        from ..parallel.flat_ddp import FlatDDP
        from .accumulation import micro_batch_plan

        backend = "nccl" if self.dev.type == "cuda" else "gloo"
        # CUDA: forward + backward are replayed as one CUDA graph (the step of the small networks is launch bound: MNIST
        # CNN 1.4 ms of mostly gaps), the flat gradient buffer is reduced by one collective after it
        self.use_graph = self.dev.type == "cuda" and not self.args.no_graph
        if self.ddp is None:
            self.ddp = FlatDDP(self.module, group=group, backend=backend, lr=self.args.lr,
                               optimizer="adamw" if self.name != "mlp" else "sgd", overlap=not self.use_graph)
        else:  # re-bind after a re-rendezvous: keep buffers, rebuild the reducer for the new group
            from ..parallel.ddp import BucketAllReducer

            self.ddp.group = group
            self.ddp.world = dist.get_world_size(group) if dist.is_initialized() else 1
            self.ddp.reducer = BucketAllReducer(self.ddp.g32, self.ddp.buckets, group, backend, 0) \
                if self.ddp.world > 1 else None
            if self.ddp.reducer is not None and self.ddp.overlap and not getattr(self.ddp, "_hooked", False):
                for idx, p in enumerate(self.ddp.params):
                    p.register_post_accumulate_grad_hook(self.ddp._make_hook(idx))
        self.ddp._hooked = self.ddp.reducer is not None or getattr(self.ddp, "_hooked", False)
        world = self.ddp.world
        rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.plan = micro_batch_plan(0 if warm_up else getattr(self.args, "global_batch", 0), self.batch, world, rank)
        self.ddp.k = self.plan.k

    def _fwd_bwd(self) -> torch.Tensor:
        if self.dev.type == "cuda":
            with torch.autocast("cuda", dtype=torch.bfloat16):
                loss = torch.nn.functional.cross_entropy(self.module(self.x_dev), self.y_dev)
        else:
            loss = torch.nn.functional.cross_entropy(self.module(self.x_dev), self.y_dev)
        loss.backward()
        return loss

    def _capture(self) -> None:
        """Forward + backward of the fixed-shape step as one CUDA graph: static inputs (x_dev / y_dev), gradients
        accumulated in place into the flat buffer the parameters' ``.grad`` already point into."""
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(3):
                self._fwd_bwd()
                self.ddp.g32.zero_()
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        try:
            with torch.cuda.graph(g):
                self._graph_loss = self._fwd_bwd().detach()
            self.ddp.g32.zero_()
            self.graph = g
        except Exception as e:  # noqa: BLE001 - eager fallback (and the per-bucket overlap is gone: one all-reduce)
            self.graph_error = f"{type(e).__name__}: {e}"
            self.graph = None
            self.use_graph = False
            torch.cuda.synchronize()

    def _batch(self, j: int):
        """Synthetic inputs of micro-batch ``j``.  With a fixed global batch micro-batch j of step s takes batch s*k + j
        of the cycle, so the job's batches do not depend on the world size; otherwise each rank cycles its own."""
        if self.plan.fixed:
            return self.batches[(self._steps * self.plan.k + j) % len(self.batches)]
        b = self.batches[self.i % len(self.batches)]
        self.i += 1
        return b

    def train_step(self) -> float:
        """One optimizer step over this rank's micro-batches (one without ``--global-batch``): forward + backward of each
        adds into the flat gradient buffer -- the bucket hooks held back until the last one -- then one gradient
        reduction and one optimizer sweep.  A rank without micro-batches reduces its zero buffer."""
        n = self.plan.n
        loss_sum = None
        for j, mb in enumerate(self.plan.micro):
            x, y = self._batch(mb)
            self.x_dev.copy_(x, non_blocking=True)
            self.y_dev.copy_(y, non_blocking=True)
            if self.use_graph and self.graph is None and self.graph_error is None:
                self._capture()
            self.ddp.sync = j == n - 1
            try:
                if self.graph is not None:
                    self.graph.replay()
                    loss = self._graph_loss
                else:
                    loss = self._fwd_bwd()
            finally:
                self.ddp.sync = True
            loss = loss.detach().float()
            loss_sum = loss if loss_sum is None else loss_sum + loss
            if n > 1:
                heartbeat()               # a long accumulated step must not look like a hang to the agent
        self.ddp.finish_backward()
        self.ddp.step()
        self._steps += 1
        if loss_sum is None:
            return float("nan")
        self.loss_host.copy_(loss_sum.reshape(1), non_blocking=True)
        if self.dev.type == "cuda":
            torch.cuda.current_stream().synchronize()
        return float(self.loss_host[0]) / n

    def discard_step(self) -> None:
        if self.ddp is not None:
            self.ddp.discard_step()        # .grad are views of the flat buffer it zeroes

    def prepare_state(self) -> None:
        return                             # every rank holds the whole state

    def state_tensors(self) -> List[torch.Tensor]:
        return self.ddp.state_tensors()

    def after_state_load(self) -> None:
        return

    @property
    def step_count(self) -> int:
        return self._steps

    @step_count.setter
    def step_count(self, v: int) -> None:
        self._steps = v
        if self.ddp is not None:
            self.ddp.step_count = v

    def launches_per_step(self) -> int:
        return 1 if self.dev.type == "cuda" else 0

    gradient_sync = "flat buffer all-reduce (nccl / gloo)"

    def graph_report(self, world: int) -> Dict[str, Any]:
        """The result's CUDA-graph and all-reduce fields."""
        return {"cuda_graph": bool(self.graph), "graph_segments": None, "graph_error": self.graph_error,
                "allreduce": "nccl" if world > 1 else "none"}


def build_adapter(args, device: torch.device):
    if args.model in (*GPT2_MODELS, "bert", "bert-tiny"):
        if device.type != "cuda":
            raise RuntimeError(f"model {args.model} needs a CUDA device (hand-written sm_90a kernels)")
        return EngineAdapter(args.model, args.batch, args.seq, args)
    return TorchAdapter(args.model, args.batch, args, device)


# ------------------------------------------------------------------------------------ checkpoint
def ckpt_path(args) -> str:
    d = args.ckpt_dir or os.path.join(os.environ.get("AITJ_WORKDIR", "/tmp"), "ckpt")
    os.makedirs(d, exist_ok=True)
    job = os.environ.get("TRAININGJOB_NAME", "job")
    # per job *object*, not per name: a job submitted again under the same name must never resume from its predecessor's
    # state (the uid survives every restart of the job's replicas, which is what a checkpoint is for)
    uid = os.environ.get("AITJ_JOB_UID", "")[:8]
    return os.path.join(d, f"{job}-{uid}.pt" if uid else f"{job}.pt")


_CKPT: Dict[str, Any] = {}


def checkpointer(args):
    """The process-wide asynchronous checkpoint writer (``runtime/checkpoint.py``)."""
    from .checkpoint import AsyncCheckpointer

    path = ckpt_path(args)
    if _CKPT.get("path") != path:
        _CKPT["path"], _CKPT["writer"] = path, AsyncCheckpointer(path)
    return _CKPT["writer"]


def save_checkpoint(args, adapter, step: int) -> None:
    """Snapshot the state in stream order and write it in the background; ``AITJ_CKPT_ASYNC=0`` waits for the file."""
    w = checkpointer(args)
    extra = {"data_position": int(adapter.data_position)} if hasattr(adapter, "data_position") else None
    w.save(step, adapter.state_tensors(), extra=extra)
    if os.environ.get("AITJ_CKPT_ASYNC", "1") == "0":
        w.wait()


def load_checkpoint(args, adapter) -> int:
    from .checkpoint import load_into

    if _CKPT.get("writer") is not None:
        _CKPT["writer"].wait()              # our own write in flight (in-place recovery falls back to it)
    meta = load_into(ckpt_path(args), adapter.state_tensors())
    if meta is None:
        return 0
    adapter.after_state_load()
    if hasattr(adapter, "data_position"):
        adapter.data_position = int(meta.get("data_position", 0))
    return int(meta["step"])


# ------------------------------------------------------------------------------------ main loop
def dump_outputs(out_dir: str, adapter, losses) -> None:
    """What the timed steps computed, so that two builds can be compared output for output on the same seeded inputs:
    ``losses.npy`` (float64, the loss of every timed step, the last one being the final step's) and ``weights_sample.npy``
    (float32, 4 Mi elements of the fp32 master weights after the last step -- the state the step updates -- at indices
    drawn from a fixed seed; all of them when the model is smaller).  With several ranks the caller first gathers the
    whole state on every rank (``adapter.prepare_state()``), so the sample covers every rank's optimizer shard."""
    import numpy as np

    os.makedirs(out_dir, exist_ok=True)
    np.save(os.path.join(out_dir, "losses.npy"), np.asarray(losses, dtype=np.float64))
    w = adapter.state_tensors()[0].detach().reshape(-1)
    n = w.numel()
    if n > (1 << 22):
        idx = torch.randint(0, n, (1 << 22,), generator=torch.Generator().manual_seed(0)).sort().values
        w = w[idx.to(w.device)]
    np.save(os.path.join(out_dir, "weights_sample.npy"), w.float().cpu().numpy())


class _Left(Exception):
    """This rank is not part of the job's new world: ``run`` returns the record it carries."""


class _TimedRegion:
    """The measured steps, bracketed by barrier + synchronize and CUDA events, with the evaluations that ran inside it
    (device ms, wall ms, kernel launches) taken out of the step figures."""

    def __init__(self, use_cuda: bool):
        self.use_cuda = use_cuda
        self.from_step = -1          # first step inside the region (-1: not armed yet)
        self.eval_ms = self.eval_wall_ms = 0.0
        self.eval_launches = 0

    def arm(self, step: int, world: int) -> None:
        if world > 1:
            dist.barrier()
        if self.use_cuda:
            torch.cuda.synchronize()
            self.ev0, self.ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            self.ev0.record()
        self.t_wall0, self.t_epoch0 = time.perf_counter(), time.time()
        self.from_step = step
        self.launches0 = oplib.LAUNCHES

    def exclude(self, ms: float, wall_ms: float, launches: int) -> None:
        """An evaluation or a generation ran: out of the step figures if it was inside the region."""
        if self.from_step >= 0:
            self.eval_ms += ms
            self.eval_wall_ms += wall_ms
            self.eval_launches += launches

    def close(self, step: int, world: int, device, global_batch: int, graph_launches: int) -> Dict[str, Any]:
        """Collective, after the last step of an armed region: the timing fields of the result, the device time being
        the slowest rank's."""
        n = step - self.from_step
        if self.use_cuda:
            self.ev1.record()
            torch.cuda.synchronize()
        t_epoch1 = time.time()
        if world > 1:
            dist.barrier()
        wall_total = time.perf_counter() - self.t_wall0
        dev_ms = (self.ev0.elapsed_time(self.ev1) if self.use_cuda else wall_total * 1e3) - self.eval_ms
        wall = wall_total - self.eval_wall_ms / 1e3
        dev_ms = max_over_ranks(dev_ms, device)
        eager_launches = oplib.LAUNCHES - self.launches0 - self.eval_launches
        return {"timed_steps": n, "timed_from_step": self.from_step, "timed_region_epoch": [self.t_epoch0, t_epoch1],
                "ms_per_step": dev_ms / n, "samples_per_sec": global_batch * n / (dev_ms / 1e3),
                "wall_ms_per_step": wall * 1e3 / n,
                "gpu_launches": graph_launches * n if graph_launches else eager_launches,
                "launches_per_step": graph_launches or (eager_launches // max(1, n))}


class _Loop:
    """The training loop of one replica and the state it keeps from step to step (``run``)."""

    def __init__(self, args):
        t_proc = time.time()
        self.args = args
        self.rank = env_int("RANK", env_int("TRAININGJOB_REPLICA_INDEX", 0))
        rdv = rendezvous_from_env()
        self.world, self.port, self.generation = rdv["world"], rdv["port"], rdv["generation"]
        self.use_cuda = torch.cuda.is_available() and not args.cpu
        self.device = torch.device("cuda", env_int("LOCAL_RANK", 0) if torch.cuda.device_count() > 1 else 0) \
            if self.use_cuda else torch.device("cpu")
        if self.use_cuda:
            torch.cuda.set_device(self.device)
        if args.elastic and os.environ.get("AITJ_FAULT_TOLERANT") == "1":
            # NCCL's watchdog would take the process down on an asynchronous communicator error or a collective timeout
            # (TearDown / SkipCleanUp); a faultTolerant job handles the loss of a peer itself (StallBreaker + _recover)
            os.environ.setdefault("TORCH_NCCL_ASYNC_ERROR_HANDLING", "0")
            # A communicator that must be abortable with a peer already dead should not hold NVSwitch multicast (NVLS)
            # objects: their teardown involves every member.  Precaution, not a measured fix.  Costs the faultTolerant
            # job's all-reduce the in-switch reduction.
            os.environ.setdefault("NCCL_NVLS_ENABLE", "0")
        self.trace = {"process_start": t_proc, "torch_imported": time.time()}
        heartbeat(force=True)
        self.watcher = watcher = ElasticWatcher.from_env(self.generation)
        if watcher is not None and not args.elastic:
            watcher.poll = 5.0  # reporting only
        self.adapter = build_adapter(args, self.device)
        self.trace["model_built"] = time.time()
        heartbeat(force=True)
        self.step = 0
        self._join_job()
        # faultTolerant (types.go:47, never read by the reference): the loss of a peer is survived in place (_recover)
        self.fault_tolerant = bool(args.elastic and watcher is not None and os.environ.get("AITJ_FAULT_TOLERANT") == "1")
        self.breaker = None
        # (armed on CUDA, where a collective with a dead peer hangs instead of raising; AITJ_STALL_BREAKER=force arms it
        #  for any backend -- the CPU tests use it with collectives that are made to hang the way NCCL's do)
        hangs = self.use_cuda or os.environ.get("AITJ_STALL_BREAKER") == "force"
        if self.fault_tolerant and hangs and float(os.environ.get("AITJ_FT_ABORT_AFTER", "3")) > 0:
            self.breaker = StallBreaker(watcher, float(os.environ.get("AITJ_FT_ABORT_AFTER", "3")))
        elif watcher is not None and hangs and self.world > 1 and float(os.environ.get("AITJ_STALL_EXIT_AFTER", "3")) > 0:
            # not faultTolerant: a rank stuck behind a dead peer cannot be repaired in place; once the controller has
            # started to repair the job (newer generation) it leaves at once instead of waiting for the heartbeat time-out
            self.breaker = StallBreaker(watcher, float(os.environ.get("AITJ_STALL_EXIT_AFTER", "3")), action="exit")
        self.stopping = False
        signal.signal(signal.SIGTERM, lambda *_: setattr(self, "stopping", True))
        self.total = args.warmup + args.steps if args.steps > 0 else 1 << 60
        self.losses, self.rescales, self.recoveries = [], [], []
        # armed at the first step boundary at or past the warm-up: a replica resumed from a checkpoint (or an elastic
        # joiner) starts past `--warmup` and still gets a timed region (and counts the steps it timed)
        self.region = _TimedRegion(self.use_cuda)
        self.pending_rescale: Optional[Dict[str, Any]] = None
        # rank 0 publishes its wall-clock throughput every AITJ_REPORT_EVERY seconds (0 = only the final, device-timed
        # result), without the evaluation wall time since the last report
        self.report_every = float(os.environ.get("AITJ_REPORT_EVERY", "10"))
        self.live_t0, self.live_step0, self.live_eval_s = time.time(), self.step, 0.0
        # held-out evaluation (--eval-data): at the boundary before every step that is a multiple of --eval-every, and
        # once after the last step.  A boundary's evaluation is done once it has completed.  Every (re-)bind to a new
        # generation forgets that (last_eval_step = -1): a joiner knows nothing of it, so after a rescale or a recovery at
        # a boundary that was already evaluated -- a peer lost in the step right after an evaluation -- every rank of the
        # new generation evaluates it again, and all of them issue the same collectives.
        self.evals: List[Dict[str, Any]] = []
        self.last_eval_step = -1
        # text generation (--generate-every): at the same boundaries, after the evaluation; local to each rank, so a
        # boundary is generated once per process whatever happens to the group around it
        self.generations: List[Dict[str, Any]] = []
        self.last_generate_step = -1
        # HellaSwag (--hellaswag): at the same boundaries, after the evaluation and before the generation; collective,
        # so a (re-)bind forgets which boundary was scored, exactly as for the evaluation
        self.hellaswag: List[Dict[str, Any]] = []
        self.last_hellaswag_step = -1

    def _join_job(self) -> None:
        """Join the job's process group and take its state, and with it the loop step to start at."""
        args, adapter, rank = self.args, self.adapter, self.rank
        joiner = bool(args.elastic and self.watcher is not None and self.generation > 1 and self.world > 1)
        if joiner:
            # Joining a running job: do everything that needs no peer first -- CUDA context, model build, two throw-away
            # steps (kernel loading, cuDNN plans, allocator growth; the state is overwritten by rank 0's broadcast
            # anyway) -- and only then tell the survivors, who keep training until this rank is ready to rendezvous.
            adapter.bind(None, warm_up=True)     # single-micro-batch steps: not 2k micro-batches of throw-away work
            for _ in range(2):
                adapter.train_step()
            if self.use_cuda:
                torch.cuda.synchronize()
            t = self.trace
            t["prewarmed"] = time.time()
            self.watcher.announce_ready(rank, self.generation)
            self._log(f"joiner ready for generation {self.generation} after {t['prewarmed'] - t['process_start']:.2f}s "
                      f"of local set-up (model build {t['model_built'] - t['process_start']:.2f}s, warm-up steps "
                      f"{t['prewarmed'] - t['model_built']:.2f}s)")
        if self.world > 1:
            self._rendezvous()
            if self.watcher is not None:
                self.watcher.adopted(self.generation, self.world)
        self.trace["rendezvous_done"] = time.time()
        heartbeat(force=True)
        adapter.bind(None)
        self._log(f"world {self.world}: gradient sync = {adapter.gradient_sync}")
        restart_count = env_int("TRAININGJOB_REPLICA_RESTARTCOUNT", 0)
        start_step = 0
        if restart_count > 0 and args.ckpt_every > 0:
            start_step = load_checkpoint(args, adapter)
            adapter.step_count = start_step
            self._log(f"restart #{restart_count}: resumed from checkpoint at step {start_step}"
                      + (f", data position {adapter.data_position}" if hasattr(adapter, "data_position") else ""))
        # a joiner without a checkpoint only has its throw-away warm-up state: it must never be elected as the source
        self.step = sync_state(adapter, start_step, self.device, have_state=not joiner or start_step > 0)
        if joiner:
            self._log(f"joined generation {self.generation} (world {self.world}) at step {self.step}")

    def _log(self, message: str) -> None:
        print(f"[worker {self.rank}] {message}", flush=True)

    def _leave(self, message: str) -> None:
        self._log(message)
        raise _Left({"left": True, "generation": self.generation, "step": self.step})

    def _rendezvous(self) -> None:
        """Form the group of generation ``self.generation`` -- or of a newer one the job has moved on to meanwhile."""
        got = rendezvous(self.rank, {"generation": self.generation, "world": self.world, "port": self.port}, self.device,
                         self.watcher)
        if got is None:
            self._leave("not part of the current world any more, leaving")
        self.generation, self.world, self.port = got["generation"], got["world"], got["port"]

    def _enter(self, target: Dict[str, Any], t0: float, observed_at: float, recovered_from: Optional[str] = None,
               aborted: bool = False) -> None:
        """Move to rendezvous generation ``target`` once the old group is gone: rendezvous, re-bind the trainer, hand the
        state off; the change is timed until the first step at the new world size completes (``_rescaled``).  A rank
        outside the new world leaves.  A failed hand-off raises after a rescale, so the loop's recovery takes it over."""
        self.generation, self.world, self.port = target["generation"], target["world"], target["port"]
        if self.rank >= self.world:
            self._leave(f"leaving: world shrinks to {self.world} (generation {self.generation})")
        t1 = time.time()
        if self.world > 1 or recovered_from is not None:    # a recovery re-reads the job even for a world of one
            self._rendezvous()
        t2 = time.time()
        if aborted and self.args.ckpt_every > 0 and os.path.exists(ckpt_path(self.args)):
            # kernels released by an abort ran on with whatever the dead peer left in the buffers: do not trust this
            # rank's copy when there is a checkpoint to fall back to
            self.step = load_checkpoint(self.args, self.adapter)
            self.adapter.step_count = self.step
        if self.breaker is not None:
            self.breaker.tripped = False
            self.breaker.progress(self.generation)
        self.adapter.bind(None)
        self.last_eval_step = self.last_hellaswag_step = -1
        try:
            with guarded(self.breaker, "the state hand-off", self.generation):
                self.step = sync_state(self.adapter, self.step, self.device)
        except RuntimeError as e:
            if recovered_from is None:
                raise
            # the hand-off is a chain of collectives on the new group: ANOTHER peer died under it.  The group is gone
            # again; the step boundary's generation agreement finds the newest record and joins it through a rescale.
            self._log(f"another peer was lost during the state hand-off of generation {self.generation} "
                      f"({type(e).__name__}); joining the next generation")
            teardown_group(broken=True)
            if self.breaker is not None:
                self.breaker.tripped = False
            return
        heartbeat(force=True)
        self.watcher.adopted(self.generation, self.world)
        self.pending_rescale = {"generation": self.generation, "world": self.world, "t0": t0, "observed_at": observed_at,
                                "teardown_s": t1 - t0, "init_pg_s": t2 - t1, "sync_state_s": time.time() - t2}
        if recovered_from is not None:
            self.pending_rescale["recovered_from"] = recovered_from

    def _rescale(self) -> bool:
        """Elastic: agree on the newest rendezvous generation at the step boundary and move to it (True)."""
        if self.watcher is None or not self.args.elastic:
            return False
        target = self.watcher.agree(self.device, guard=self.breaker)
        if target is None or target["generation"] == self.generation:
            return False
        t0 = time.time()
        self._log(f"rendezvous generation {self.generation} -> {target['generation']} "
                  f"(world {self.world} -> {target['world']}) at step {self.step}")
        if dist.is_initialized():
            self.adapter.prepare_state()       # sharded optimizer state -> whole state on every survivor
            if self.use_cuda:
                torch.cuda.synchronize()
            dist.destroy_process_group()
        self._enter(target, t0, target.get("observed_at", t0))
        return True

    def _recover(self, failure) -> None:
        """faultTolerant: a peer died under a collective.  (gloo raises in the survivors; for NCCL the StallBreaker aborts
        the communicator.)  The survivors keep their process, device state and -- on GPUs -- CUDA context: drop the
        broken group, wait for the controller to replace the lost replica (restart scope Pod, new rendezvous
        generation), re-rendezvous and continue from the survivors' state."""
        t0 = time.time()
        aborted = self.breaker is not None and self.breaker.tripped
        self._log(f"step {self.step}: lost a peer ({failure[0]}: {failure[1]}); keeping state, waiting for the next "
                  f"rendezvous generation")
        # pending work handles keep the group's sockets open; a peer that is blocked on *us* (gloo does not
        # propagate a failure beyond the dead rank's direct neighbours) only errors out once they really close
        self.adapter.discard_step()
        teardown_group(broken=True)
        gc.collect()
        target = wait_for_newer_generation(self.watcher, self.generation, float(os.environ.get("AITJ_FT_WAIT", "120")),
                                           should_stop=lambda: self.stopping)
        if target is None and self.stopping:
            self._log("terminated while waiting for the job to be repaired")
            return
        if target is None:
            self._log("no new rendezvous generation was published: giving up")
            raise RuntimeError(f"collective failed and the job was not repaired: {failure[0]}: {failure[1]}")
        self._enter(target, t0, t0, recovered_from=failure[0], aborted=aborted)

    def _eval_due(self) -> bool:
        s, a = self.step, self.args
        return hasattr(self.adapter, "eval_data") and s != self.last_eval_step and \
            ((s > 0 and a.eval_every > 0 and s % a.eval_every == 0) or (a.steps > 0 and s >= self.total))

    def _off_the_clock(self, what: str, work):
        """Run ``work(progress)`` -- an evaluation or a generation -- under the stall breaker, and take its device time,
        wall time and kernel launches out of the step figures.  Returns (its result, device ms)."""
        t0 = time.perf_counter()
        launches_before = oplib.LAUNCHES
        if self.use_cuda:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
        with guarded(self.breaker, what, self.generation):
            # as long as its pieces make it: the stall breaker sees progress after each one, not the patience of a
            # single training step for the whole of it
            out = work(None if self.breaker is None else lambda: self.breaker.progress(self.generation))
        wall_ms = (time.perf_counter() - t0) * 1e3
        if self.use_cuda:
            e1.record()
            e1.synchronize()
        ms = e0.elapsed_time(e1) if self.use_cuda else wall_ms
        self.region.exclude(ms, wall_ms, oplib.LAUNCHES - launches_before)
        self.live_eval_s += wall_ms / 1e3
        return out, ms

    def _hellaswag_due(self) -> bool:
        s, a = self.step, self.args
        return hasattr(self.adapter, "hellaswag") and s != self.last_hellaswag_step and \
            ((s > 0 and a.hellaswag_every > 0 and s % a.hellaswag_every == 0) or (a.steps > 0 and s >= self.total))

    def _score(self) -> None:
        rec, ms = self._off_the_clock("a HellaSwag scoring", lambda progress: self.adapter.score(progress=progress))
        rec = dict(step=self.step, **rec, ms=round(ms, 3))
        self.hellaswag.append(rec)
        self.last_hellaswag_step = self.step
        if self.rank == 0:
            self._log(f"step {self.step}: hellaswag acc {rec['acc']:.4f} ({rec['correct']}/{rec['examples']}) in "
                      f"{ms:.1f} ms")

    def _generate_due(self) -> bool:
        s, a = self.step, self.args
        every = getattr(a, "generate_every", None)
        return every is not None and hasattr(self.adapter, "generator") and s != self.last_generate_step and \
            ((s > 0 and every > 0 and s % every == 0) or (a.steps > 0 and s >= self.total))

    def _generate(self) -> None:
        rec, ms = self._off_the_clock("a generation", lambda progress: self.adapter.generate(self.step, progress))
        rec = dict(step=self.step, ms=round(ms, 3), **rec)
        self.generations.append(rec)
        self.last_generate_step = self.step
        if self.rank == 0:
            self._log(f"step {self.step}: generated {len(rec['tokens'])} sequences of {len(rec['tokens'][0])} tokens "
                      f"in {ms:.1f} ms (seed {rec['seed']})")
            for i, seq in enumerate(rec.get("text") or rec["tokens"]):
                self._log(f"step {self.step}: generation {i}: {seq!r}" if "text" in rec else
                          f"step {self.step}: generation {i}: {' '.join(map(str, seq))}")

    def _evaluate(self) -> None:
        rec, ms = self._off_the_clock("an evaluation", lambda progress: self.adapter.evaluate(progress=progress))
        rec = {"step": self.step, "loss": rec["loss"], "tokens": rec["tokens"], "samples": rec["samples"],
               "ms": round(ms, 3)}
        self.evals.append(rec)
        self.last_eval_step = self.step
        if self.rank == 0:
            self._log(f"step {self.step}: eval loss {rec['loss']:.6f} over {rec['samples']} held-out windows "
                      f"({rec['tokens']} tokens) in {ms:.1f} ms")

    def run(self) -> Dict[str, Any]:
        while (self.step < self.total or self._eval_due() or self._hellaswag_due() or self._generate_due()) and \
                not self.stopping:
            if self.breaker is not None:
                self.breaker.progress(self.generation)
                # patience from this generation's completed steps: the first step on a freshly bound trainer captures
                # CUDA graphs / loads kernels, and an accumulated step can take seconds -- neither is a stall
                self.breaker.begin_step(self.generation)
            failure = None
            try:
                if self._rescale():
                    continue    # back to the step boundary: every rank (joiners included) runs the same sequence
                if self.region.from_step < 0 and self.step >= self.args.warmup and self.args.steps > 0:
                    self.region.arm(self.step, self.world)
                if self._eval_due():
                    self._evaluate()
                if self._hellaswag_due():
                    self._score()
                if self._generate_due():
                    self._generate()
                if self.step >= self.total:
                    continue              # the evaluation / generation after the last step: the loop ends here
                with guarded(self.breaker, "this step", self.generation):
                    t_step = time.perf_counter()
                    loss = self.adapter.train_step()
                    if self.breaker is not None:
                        self.breaker.step_done(self.generation, time.perf_counter() - t_step)
            except RuntimeError as e:
                # Without faultTolerant the error ends this replica and the job's restartPolicy / restartScope take
                # over, as in the reference (pod.go:208-250).
                if not self.fault_tolerant or self.world <= 1:
                    raise
                failure = (type(e).__name__, (str(e).splitlines() or [""])[0][:160])
            if failure is not None:
                # (outside the except block: the traceback of the failed step references the work handles of the broken
                # group, and with them its sockets)
                self._recover(failure)
                continue
            self._step_done(loss)
        return self._finish()

    def _step_done(self, loss: float) -> None:
        self.losses.append(loss)
        self.step += 1
        heartbeat()
        if self.pending_rescale is not None:
            self._rescaled()
        if "first_step_done" not in self.trace:
            self.trace["first_step_done"] = time.time()
            if self.watcher is not None:
                self.watcher.report_trace(self.rank, self.trace)
        if self.rank == 0 and self.watcher is not None and self.report_every > 0 and \
                time.time() - self.live_t0 >= self.report_every:
            self._report_live()
        if self.args.ckpt_every > 0 and self.step % self.args.ckpt_every == 0:
            self.adapter.prepare_state()
            if self.rank == 0:
                save_checkpoint(self.args, self.adapter, self.adapter.step_count)
        if self.args.step_sleep > 0:
            time.sleep(self.args.step_sleep)

    def _rescaled(self) -> None:
        """The first completed step at the new world size ends the rescale."""
        p, now = self.pending_rescale, time.time()
        rec = {"generation": p["generation"], "world": p["world"], "seconds": now - p["t0"],
               "since_change": now - p["observed_at"], "teardown_s": round(p["teardown_s"], 4),
               "init_pg_s": round(p["init_pg_s"], 4), "sync_state_s": round(p["sync_state_s"], 4)}
        rec["first_step_s"] = round(rec["seconds"] - rec["teardown_s"] - rec["init_pg_s"] - rec["sync_state_s"], 4)
        if "recovered_from" in p:
            rec["recovered_from"] = p["recovered_from"]
            self.recoveries.append(rec)
        self.rescales.append(rec)
        self._log(f"step {self.step}: rescaled to world={rec['world']} gen={rec['generation']} in {rec['seconds']:.3f}s")
        if self.watcher is not None:
            self.watcher.report_rescale(self.rank, rec, force="recovered_from" in rec)   # rank 0 may be the replaced one
        self.pending_rescale = None

    def _report_live(self) -> None:
        dt, n = time.time() - self.live_t0 - self.live_eval_s, self.step - self.live_step0
        if n > 0 and dt > 0:
            G = self.adapter.plan.global_batch
            live = {"samples_per_sec": round(G * n / dt, 2), "ms_per_step": round(dt * 1e3 / n, 3), "world": self.world,
                    "steps_done": self.step, "global_batch": G, "recoveries": len(self.recoveries)}
            if self.evals:
                live.update(eval_loss=self.evals[-1]["loss"], eval_step=self.evals[-1]["step"])
            if self.hellaswag:
                live.update(hellaswag_acc=self.hellaswag[-1]["acc"], hellaswag_step=self.hellaswag[-1]["step"])
            self.watcher.report_live(self.rank, live)
        self.live_t0, self.live_step0, self.live_eval_s = time.time(), self.step, 0.0

    def _finish(self) -> Dict[str, Any]:
        args, adapter, losses, rank = self.args, self.adapter, self.losses, self.rank
        result: Dict[str, Any] = {"rank": rank, "world": self.world, "steps_done": self.step,
                                  "generation": self.generation, "final_loss": losses[-1] if losses else None,
                                  "rescales": self.rescales, "recoveries": self.recoveries, "trace": self.trace}
        if hasattr(adapter, "data_position"):
            result["data_position"] = adapter.data_position
        if hasattr(adapter, "eval_data"):
            result.update(evals=self.evals, eval_loss_last=self.evals[-1]["loss"] if self.evals else None)
        if hasattr(adapter, "hellaswag"):
            result.update(hellaswag=self.hellaswag,
                          hellaswag_acc_last=self.hellaswag[-1]["acc"] if self.hellaswag else None)
        if hasattr(adapter, "generator"):
            result["generations"] = self.generations
        if self.breaker is not None:
            self.breaker.stop()
        if _CKPT.get("writer") is not None:
            _CKPT["writer"].wait(60.0)
        n_timed = self.step - self.region.from_step if self.region.from_step >= 0 else 0
        if args.steps > 0 and self.step >= self.total and n_timed > 0:
            plan = adapter.plan
            result.update(self.region.close(self.step, self.world, self.device, plan.global_batch,
                                            adapter.launches_per_step()))
            result.update({
                "global_batch": plan.global_batch, "batch_per_gpu": args.batch,
                "micro_batches": plan.k, "micro_batches_this_rank": plan.n,
                "h2d_bytes_per_step": adapter.h2d_bytes, "d2h_bytes_per_step": adapter.d2h_bytes,
                "loss_first": losses[0] if losses else None, "loss_last": losses[-1] if losses else None,
                "flops_per_step": getattr(adapter, "flops_per_step", 0.0) * plan.n,     # this rank's work
                "describe": adapter.describe,
            })
            result.update(adapter.graph_report(self.world))
        if args.dump_outputs and n_timed > 0:
            # collective: with the owner-sharded optimizer each rank keeps only its own range of the master weights current
            adapter.prepare_state()
            if rank == 0:
                dump_outputs(args.dump_outputs, adapter, losses[-n_timed:])
        if rank == 0 and args.result:
            os.makedirs(os.path.dirname(os.path.abspath(args.result)), exist_ok=True)
            with open(args.result + ".tmp", "w") as f:
                json.dump(result, f)
            os.replace(args.result + ".tmp", args.result)
        if rank == 0 and self.watcher is not None:
            self.watcher.report_result(result)
        if dist.is_initialized():
            try:
                dist.destroy_process_group()
            except Exception:  # noqa: BLE001
                pass
        return result


def run(args) -> Dict[str, Any]:
    """One replica from start to end: the result record, or ``{"left": True, ...}`` when the job's world shrank
    below this rank."""
    try:
        return _Loop(args).run()
    except _Left as left:
        return left.args[0]


def parse_args(argv=None):
    ap = argparse.ArgumentParser(prog="aitj-worker")
    ap.add_argument("--model", default="gpt2",
                    choices=[*GPT2_MODELS, "bert", "bert-tiny", "resnet50", "mnist", "mlp"])
    ap.add_argument("--batch", type=int, default=16, help="per-GPU batch size")
    ap.add_argument("--seq", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=20, help="timed steps (0 = run until SIGTERM)")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--lr", type=float, default=3e-4)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--gemm", default="wgmma", choices=["wgmma", "cublas"])
    ap.add_argument("--no-graph", action="store_true")
    ap.add_argument("--cpu", action="store_true")
    ap.add_argument("--elastic", action="store_true")
    ap.add_argument("--result", default="")
    ap.add_argument("--dump-outputs", default="", metavar="DIR",
                    help="after the timed steps, write what they computed to DIR/*.npy (see dump_outputs)")
    ap.add_argument("--ckpt-dir", default="")
    ap.add_argument("--ckpt-every", type=int, default=0)
    ap.add_argument("--step-sleep", type=float, default=0.0)
    ap.add_argument("--data", default="", metavar="PATH_OR_GLOB",
                    help="train on these token shards (llm.c .bin shards or raw uint16 files; GPT-2 models) instead of "
                         "synthetic tokens")
    ap.add_argument("--doc-mask", action="store_true",
                    help="with --data: a token attends only to earlier tokens of its own document (documents start at "
                         "the end-of-text token); runs the wgmma attention kernels")
    ap.add_argument("--eot-token", type=int, default=50256, help="end-of-text token id that starts a document")
    ap.add_argument("--global-batch", type=int, default=0, metavar="G",
                    help="samples per optimizer step for the whole job, at any world size: each step trains G / --batch "
                         "micro-batches, spread over the ranks, and sums their gradients (0 = world size x --batch)")
    ap.add_argument("--eval-data", default="", metavar="PATH_OR_GLOB",
                    help="evaluate on these held-out token shards (formats as --data; GPT-2 models, wgmma GEMMs)")
    ap.add_argument("--eval-samples", type=int, default=0, metavar="S",
                    help="held-out windows per evaluation, the first S of the stream (0 = 20 x --batch)")
    ap.add_argument("--eval-every", type=int, default=0, metavar="N",
                    help="evaluate before every step that is a multiple of N, and after the last step (0 = only after "
                         "the last step)")
    ap.add_argument("--hellaswag", default="", metavar="PATH",
                    help="score HellaSwag from this llm.c eval file (dev/data/hellaswag.py; GPT-2 models, wgmma GEMMs, "
                         "--seq a multiple of 128)")
    ap.add_argument("--hellaswag-every", type=int, default=None, metavar="N",
                    help="score HellaSwag before every step that is a multiple of N, and after the last step (0 = only "
                         "after the last step)")
    # text generation (GPT-2): "generate", because "samples" already names data windows here
    ap.add_argument("--generate-every", type=int, default=None, metavar="N",
                    help="generate text before every step that is a multiple of N, and after the last step (0 = only "
                         "after the last step)")
    ap.add_argument("--generate-count", type=int, default=None, metavar="S", help="sequences per generation (4)")
    ap.add_argument("--generate-tokens", type=int, default=None, metavar="K", help="new tokens per sequence (64)")
    ap.add_argument("--generate-prompt", default=None, metavar="IDS",
                    help="comma-separated prompt token ids (default: --eot-token)")
    ap.add_argument("--temperature", type=float, default=None, help="sampling temperature, 0 = greedy (1.0)")
    ap.add_argument("--top-k", type=int, default=None, help="sample among the K most likely tokens (0 = all)")
    ap.add_argument("--tokenizer", default=None, metavar="PATH",
                    help="an llm.c gpt2_tokenizer.bin: generations are also reported as text")
    args = ap.parse_args(argv)
    _check_generation_args(ap, args)
    if args.eval_data and args.model not in GPT2_MODELS:
        ap.error(f"--eval-data evaluates GPT-2 models only, not {args.model}")
    if args.eval_data and args.gemm != "wgmma":
        ap.error("--eval-data needs --gemm wgmma: the evaluation loss is computed in the wgmma logits GEMM's epilogue")
    if args.eval_samples < 0 or args.eval_every < 0:
        ap.error("--eval-samples and --eval-every cannot be negative")
    if (args.eval_samples or args.eval_every) and not args.eval_data:
        ap.error("--eval-samples and --eval-every need --eval-data")
    _check_hellaswag_args(ap, args)
    if args.global_batch < 0 or args.global_batch % args.batch:
        ap.error(f"--global-batch {args.global_batch} is not a multiple of --batch {args.batch}")
    if args.global_batch and os.environ.get("AITJ_ALLREDUCE") == "mc":
        ap.error("--global-batch cannot be used with AITJ_ALLREDUCE=mc: the multicast gradient path has no micro-batch "
                 "accumulation")
    if args.doc_mask and not args.data:
        ap.error("--doc-mask needs --data")
    if args.data and args.model not in GPT2_MODELS:
        ap.error(f"--data trains GPT-2 models only, not {args.model}")
    if args.data:
        vocab = GPT2_MODELS[args.model].vocab_size
        if args.doc_mask and not 0 <= args.eot_token < vocab:
            ap.error(f"--eot-token {args.eot_token} is outside the vocabulary of {args.model} (size {vocab})")
    return args


def _check_hellaswag_args(ap, args) -> None:
    if args.hellaswag_every is not None and not args.hellaswag:
        ap.error("--hellaswag-every needs --hellaswag")
    args.hellaswag_every = args.hellaswag_every or 0
    if not args.hellaswag:
        return
    if args.model not in GPT2_MODELS:
        ap.error(f"--hellaswag scores GPT-2 models only, not {args.model}")
    if args.gemm != "wgmma":
        ap.error("--hellaswag needs --gemm wgmma: the completions' losses are computed in the wgmma logits GEMM's "
                 "epilogue")
    if args.seq % 128:
        ap.error(f"--hellaswag needs --seq a multiple of 128 (the document-masked attention's tile), not {args.seq}")
    if args.hellaswag_every < 0:
        ap.error("--hellaswag-every cannot be negative")


def _check_generation_args(ap, args) -> None:
    """Refuse generation flags that cannot run, and fill in the defaults of the others."""
    given = [f for f, v in (("--generate-count", args.generate_count), ("--generate-tokens", args.generate_tokens),
                            ("--generate-prompt", args.generate_prompt), ("--temperature", args.temperature),
                            ("--top-k", args.top_k), ("--tokenizer", args.tokenizer)) if v is not None]
    if args.generate_every is None:
        if given:
            ap.error(f"{', '.join(given)} need --generate-every")
        return
    if args.model not in GPT2_MODELS:
        ap.error(f"--generate-every generates from GPT-2 models only, not {args.model}")
    args.generate_count = 4 if args.generate_count is None else args.generate_count
    args.generate_tokens = 64 if args.generate_tokens is None else args.generate_tokens
    args.temperature = 1.0 if args.temperature is None else args.temperature
    args.top_k = 0 if args.top_k is None else args.top_k
    if args.generate_every < 0 or args.generate_tokens < 0 or args.top_k < 0 or not args.temperature >= 0:
        ap.error("--generate-every, --generate-tokens, --temperature and --top-k cannot be negative")
    if args.generate_count < 1:
        ap.error(f"--generate-count {args.generate_count}: generate at least one sequence")
    cfg = GPT2_MODELS[args.model]
    if args.generate_prompt is None:
        prompt = [args.eot_token]
        what = f"the default prompt, --eot-token {args.eot_token},"
    else:
        try:
            prompt = [int(t) for t in args.generate_prompt.split(",")]
        except ValueError:
            ap.error(f"--generate-prompt {args.generate_prompt!r} is not a comma-separated list of token ids")
        what = "--generate-prompt id"
    bad = [t for t in prompt if not 0 <= t < cfg.vocab_size]
    if bad:
        ap.error(f"{what} {bad[0]} is outside the vocabulary of {args.model} (size {cfg.vocab_size})")
    args.generate_prompt = prompt
    if args.top_k > cfg.vocab_size:
        ap.error(f"--top-k {args.top_k} exceeds the vocabulary of {args.model} (size {cfg.vocab_size})")
    if len(prompt) + args.generate_tokens > cfg.block_size:
        ap.error(f"the prompt ({len(prompt)} tokens) plus --generate-tokens {args.generate_tokens} exceed the block size "
                 f"of {args.model} ({cfg.block_size})")


def main(argv=None) -> int:
    args = parse_args(argv)
    res = run(args)
    if res.get("samples_per_sec"):
        print(f"[worker {res['rank']}] {res['samples_per_sec']:.1f} samples/s  {res['ms_per_step']:.3f} ms/step "
              f"loss {res.get('loss_first')} -> {res.get('loss_last')}", flush=True)
    return 0


def _record_exit(code: int) -> None:
    """``$AITJ_EXIT_FILE``: lets an agent that adopted this process after a restart (and therefore cannot wait() for
    it) still learn how it ended."""
    path = os.environ.get("AITJ_EXIT_FILE", "")
    if not path:
        return
    try:
        with open(path, "w") as f:
            f.write(str(int(code)))
    except OSError:
        pass


def cli() -> None:
    """Process entry point (``python -m ...runtime.worker`` and the ``aitj-worker`` script): runs ``main`` and records the
    exit code in ``$AITJ_EXIT_FILE`` however it ends."""
    try:
        code = main()
    except SystemExit as e:
        code = e.code if isinstance(e.code, int) else (0 if e.code is None else 1)
        _record_exit(code)
        raise
    except BaseException:
        _record_exit(1)
        raise
    _record_exit(code)
    sys.exit(code)


if __name__ == "__main__":
    cli()
