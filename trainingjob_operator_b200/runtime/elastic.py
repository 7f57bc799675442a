"""Worker-side elastic agent: follow ``status.rendezvous`` of the owning AITrainingJob.

The reference declares ``minReplicas`` / ``maxReplicas`` / ``edlPolicy`` but delegates membership
changes to an external Paddle EDL runtime (SURVEY.md §0.3, §2.4 "Elastic DP").  Here the controller
publishes a rendezvous *generation* (``controller/elastic.py``) and every worker runs this watcher:
a side thread polls the job object on the API server (``AITJ_MASTER``); at each step boundary the
ranks agree -- one tiny MAX all-reduce -- on the newest generation any of them has seen, so they all
leave the old process group at the same step.  The watcher also reports lifecycle timestamps and the
final metrics back onto the job (annotations), which is how reconcile->first-step and rescale latency
are measured end to end.
"""
from __future__ import annotations

import json
import os
import threading
import time
from typing import Any, Dict, Optional

import torch
import torch.distributed as dist

from .rendezvous import guarded

ANN_METRICS = "aitj.b200/metrics"
ANN_WORKER_TRACE = "aitj.b200/worker-trace"
ANN_RESCALE = "aitj.b200/rescale-trace"
ANN_READY_PREFIX = "aitj.b200/ready-r"     # + rank: the generation that rank has finished its local set-up for


def env_int(name: str, default: int = 0) -> int:
    try:
        return int(os.environ.get(name, default))
    except (TypeError, ValueError):
        return default


def rendezvous_from_env() -> Dict[str, int]:
    return {"world": env_int("WORLD_SIZE", 1), "port": env_int("MASTER_PORT", 29500),
            "generation": env_int("AITJ_RENDEZVOUS_GENERATION", 0)}


class ElasticWatcher:
    def __init__(self, master: str, namespace: str, job: str, role: str, generation: int, poll: float = 0.1,
                 world: int = 0):
        from ..api import register as R
        from ..store.transport import HTTPTransport

        self._t = HTTPTransport(master, timeout=5.0, user_agent="aitj-worker")
        self._info = R.AITRAININGJOB
        self.ns, self.job, self.role = namespace, job, role
        self.generation = generation
        # world size this worker currently runs at: ranks >= it in a newer, larger generation are joiners, and the
        # generation is only adopted once every joiner announced that its local set-up (CUDA context, model build,
        # warm-up step) is done -- survivors keep training meanwhile instead of idling in the rendezvous
        self.world = world or env_int("WORLD_SIZE", 1)
        self.ready_timeout = float(os.environ.get("AITJ_JOIN_READY_TIMEOUT", "90"))
        self._first_seen: Dict[int, float] = {}
        self.poll = poll
        self._latest: Optional[Dict[str, Any]] = None
        self._lock = threading.Lock()
        self._stop = threading.Event()
        self._thread = threading.Thread(target=self._loop, name="elastic-watch", daemon=True)
        self._thread.start()
        self.check_every = max(1, env_int("AITJ_ELASTIC_CHECK_EVERY", 1))
        self._n = 0

    @classmethod
    def from_env(cls, generation: int) -> Optional["ElasticWatcher"]:
        master = os.environ.get("AITJ_MASTER")
        job = os.environ.get("TRAININGJOB_NAME")
        if not master or not job:
            return None
        return cls(master, os.environ.get("TRAININGJOB_NAMESPACE", "default"), job,
                   os.environ.get("TRAININGJOB_REPLICA_NAME", "trainer"), generation, world=env_int("WORLD_SIZE", 1))

    # ------------------------------------------------------------------ polling thread
    def _fetch(self) -> Optional[Dict[str, Any]]:
        try:
            obj = self._t.get(self._info, self.ns, self.job)
        except Exception:  # noqa: BLE001 - API server briefly unreachable: keep training
            return None
        rdv = (obj.get("status") or {}).get("rendezvous")
        if not rdv:
            return None
        sizes = rdv.get("worldSizes") or {}
        world = None
        for k, v in sizes.items():
            if k.lower() == self.role.lower():
                world = int(v)
        if world is None:
            return None
        ann = (obj.get("metadata") or {}).get("annotations") or {}
        ready = {}
        for k, v in ann.items():
            if k.startswith(ANN_READY_PREFIX):
                try:
                    ready[int(k[len(ANN_READY_PREFIX):])] = int(json.loads(v))
                except (TypeError, ValueError):
                    pass
        return {"generation": int(rdv.get("generation", 0)), "world": world, "port": int(rdv.get("masterPort", 0)),
                "ready": ready}

    def fetch_now(self) -> Optional[Dict[str, Any]]:
        """The job's current rendezvous record, read synchronously (no readiness gating): used while (re)joining."""
        return self._fetch()

    def _joiners_ready(self, r: Dict[str, Any]) -> bool:
        gen = r["generation"]
        first = self._first_seen.setdefault(gen, time.time())
        missing = [j for j in range(self.world, r["world"]) if r["ready"].get(j, -1) < gen]
        if not missing:
            return True
        return time.time() - first > self.ready_timeout      # a joiner that never shows up must not block forever

    def _loop(self) -> None:
        while not self._stop.wait(self.poll):
            r = self._fetch()
            if r is None:
                continue
            if r["generation"] > self.generation and not self._joiners_ready(r):
                continue
            with self._lock:
                if self._latest is None or r["generation"] > self._latest["generation"]:
                    r["observed_at"] = self._first_seen.get(r["generation"], time.time())
                    self._latest = r

    def _wait_for(self, generation: int, timeout: float = 30.0) -> Optional[Dict[str, Any]]:
        deadline = time.time() + timeout
        while time.time() < deadline:
            with self._lock:
                if self._latest is not None and self._latest["generation"] >= generation:
                    return dict(self._latest)
            time.sleep(0.01)
        return None

    # ------------------------------------------------------------------ step-boundary agreement
    def agree(self, device: torch.device, guard=None) -> Optional[Dict[str, Any]]:
        """Newest rendezvous record every current rank can adopt now, or None.  ``guard`` (the worker's StallBreaker):
        the MAX all-reduce below is a collective like any other -- a rank whose peer died after the previous step sits
        in it, so it is marked as "inside a step" for the breaker (the bounded wait for joiners that follows is not)."""
        self._n += 1
        if self._n % self.check_every:
            return None
        with self._lock:
            mine = self._latest["generation"] if self._latest else self.generation
        newest = mine
        if dist.is_initialized() and dist.get_world_size() > 1:
            t = torch.tensor([mine], dtype=torch.int64, device=device if device.type == "cuda" else "cpu")
            with guarded(guard, "the generation agreement"):
                dist.all_reduce(t, op=dist.ReduceOp.MAX)
                newest = int(t[0])
        if newest <= self.generation:
            return None
        return self._wait_for(newest)

    def adopted(self, generation: int, world: int = 0) -> None:
        self.generation = generation
        if world:
            self.world = world

    def announce_ready(self, rank: int, generation: int) -> None:
        """A joiner finished everything it can do alone; survivors may now switch to ``generation``."""
        self._annotate(f"{ANN_READY_PREFIX}{rank}", generation)

    # ------------------------------------------------------------------ reporting
    def _annotate(self, key: str, value: Any) -> None:
        try:
            self._t.patch(self._info, self.ns, self.job, {"metadata": {"annotations": {key: json.dumps(value)}}})
        except Exception:  # noqa: BLE001
            pass

    def report_trace(self, rank: int, trace: Dict[str, float]) -> None:
        if rank == 0:
            self._annotate(ANN_WORKER_TRACE, {k: round(v, 4) for k, v in trace.items()})

    def report_rescale(self, rank: int, rec: Dict[str, Any], force: bool = False) -> None:
        if rank == 0 or force:
            rec = dict(rec)
            rec["at"] = round(time.time(), 4)
            self._annotate(ANN_RESCALE, rec)

    def report_result(self, result: Dict[str, Any]) -> None:
        keep = {k: result.get(k) for k in ("samples_per_sec", "ms_per_step", "global_batch", "world", "steps_done",
                                           "loss_first", "loss_last", "gpu_launches", "cuda_graph")}
        keep["recoveries"] = len(result.get("recoveries") or [])
        if result.get("evals"):
            keep.update(eval_loss=result["evals"][-1]["loss"], eval_step=result["evals"][-1]["step"])
        if result.get("hellaswag"):
            keep.update(hellaswag_acc=result["hellaswag"][-1]["acc"], hellaswag_step=result["hellaswag"][-1]["step"])
        t = getattr(self, "_live_thread", None)
        if t is not None:
            t.join(5.0)                     # an interim report in flight must not land after (and over) the final one
        self._annotate(ANN_METRICS, keep)

    def report_live(self, rank: int, rec: Dict[str, Any]) -> None:
        """Interim throughput of a running job (``aitjctl top``, ``aitj_job_samples_per_second``): written from a
        short-lived side thread so the step loop never waits for the API server."""
        if rank != 0:
            return
        t = getattr(self, "_live_thread", None)
        if t is not None and t.is_alive():
            return                          # the previous report is still on its way: skip this one
        self._live_thread = threading.Thread(target=self._annotate, args=(ANN_METRICS, dict(rec, live=True)),
                                             daemon=True)
        self._live_thread.start()

    def stop(self) -> None:
        self._stop.set()
