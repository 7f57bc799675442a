"""All-in-one single-box control plane: API server + node agent + N (leader-elected) operators.

There is no such thing in the reference (it needs an external Kubernetes, SURVEY.md L0); on one
8xH100 machine this is the deployment unit: ``python -m trainingjob_operator_b200.cmd.local up``
starts everything in one process (or use the three binaries ``cmd.apiserver``, ``cmd.agent``,
``cmd.main`` separately -- e.g. two operators for leader fail-over).  ``LocalCluster`` is also what
tests, ``bench.py`` and ``__graft_entry__.smoke`` use as "the public API a user calls".
"""
from __future__ import annotations

import argparse
import os
import sys
import tempfile
import threading
import time
from typing import List, Optional

from ..agent.agent import NodeAgent
from ..api import constants as C
from ..api.types import AITrainingJob
from ..client.clientset import Clientset, new_for_config
from ..store.apiserver import APIError, APIServer
from ..store.http import APIHTTPServer
from ..utils import klog
from . import options as options_mod
from . import server as server_mod


class LocalCluster:
    def __init__(self, num_gpus: Optional[int] = None, workdir: Optional[str] = None, wal: bool = False,
                 operators: int = 1, leader_elect: bool = False, http: bool = True, port: int = 0,
                 option: Optional[options_mod.TrainingJobOperatorOption] = None, health_prober=None,
                 health_period: float = 1.0, verbosity: int = 0, warm_pool: int = 0, gpu_visibility: str = "pinned"):
        self.workdir = workdir or tempfile.mkdtemp(prefix="aitj-")
        os.makedirs(self.workdir, exist_ok=True)
        klog.configure(verbosity, True)
        klog.set_verbosity(verbosity)
        self.api = APIServer(os.path.join(self.workdir, "store.wal") if wal else "")
        self.http = APIHTTPServer(self.api, port=port).start() if http else None
        self.stop_event = threading.Event()
        self.clientset: Clientset = new_for_config(server=self.api)
        self._agent_kw = dict(num_gpus=num_gpus, workdir=self.workdir, health_prober=health_prober,
                              health_period=health_period, warm_pool=warm_pool, gpu_visibility=gpu_visibility)
        self.agent = NodeAgent(new_for_config(server=self.api), **self._agent_kw)
        self._agent_stop = threading.Event()
        self.option = option or options_mod.TrainingJobOperatorOption()
        self.option.master_url = self.http.url if self.http else ""
        if leader_elect:
            self.option.leader_election.leader_elect = True
        self._operators = operators
        self._op_threads: List[threading.Thread] = []
        self._op_stops: List[threading.Event] = []
        self._op_opts: list = []
        self.operator_errors: List[BaseException] = []

    @property
    def url(self) -> str:
        return self.http.url if self.http else ""

    def _start_agent(self) -> None:
        agent_stop = self._agent_stop
        threading.Thread(target=lambda: (self.stop_event.wait(), agent_stop.set()), daemon=True).start()
        self.agent.start(agent_stop)

    def restart_agent(self) -> dict:
        """Simulates an agent crash + restart: the old agent's loops stop without touching its worker processes, a fresh
        ``NodeAgent`` (new supervisor, empty in-memory state) takes over the same nodes and re-adopts what is still
        running.  Returns the new agent's recovery summary."""
        self._agent_stop.set()
        for t in list(getattr(self.agent, "_threads", [])):
            t.join(timeout=3)
        self.agent.queue.shutdown()
        self.agent._kill_zygotes()
        kw = dict(self._agent_kw)
        kw["num_gpus"] = self.agent.num_gpus
        self.agent = NodeAgent(new_for_config(server=self.api), **kw)
        self._agent_stop = threading.Event()
        seen: dict = {}
        orig = self.agent.recover
        self.agent.recover = lambda: seen.update(orig()) or seen       # capture what start() recovers
        self._start_agent()
        return seen

    def start(self) -> "LocalCluster":
        self.api.start_housekeeping(self.stop_event)       # event TTL + WAL compaction, as the stand-alone daemon does
        self._start_agent()
        for i in range(self._operators):
            self.start_operator(i)
        return self

    def start_operator(self, index: int = 0, identity: str = "") -> threading.Event:
        import copy

        opt = copy.deepcopy(self.option)
        opt.identity = identity or (f"operator-{index}" if opt.leader_election.leader_elect else "")
        op_stop = threading.Event()
        threading.Thread(target=lambda: (self.stop_event.wait(), op_stop.set()), daemon=True).start()

        def body():
            try:
                server_mod.run(opt, stop=op_stop, server=self.api, fatal_on_lost_lease=False)
            except BaseException as e:  # noqa: BLE001
                self.operator_errors.append(e)

        t = threading.Thread(target=body, name=f"operator-{index}", daemon=True)
        t.start()
        self._op_threads.append(t)
        self._op_stops.append(op_stop)
        self._op_opts.append(opt)
        return op_stop

    def stop_operator(self, index: int, crash: bool = False) -> None:
        """Stops one operator.  ``crash=True`` simulates kill -9: the lease is NOT handed over, so the standby has to
        wait for it to expire (leader fail-over tests / tools/failover_check.py)."""
        if crash:
            self._op_opts[index].crash_on_stop = True
        self._op_stops[index].set()

    # ------------------------------------------------------------------ convenience API
    def jobs(self, namespace: str = "default"):
        return self.clientset.elasticdeeplearning_v1().aitrainingjobs(namespace)

    def apply(self, obj: dict, namespace: str = "default") -> AITrainingJob:
        job = AITrainingJob.from_dict(obj)
        ns = job.namespace or namespace
        import json
        import time as _t

        job.metadata.setdefault("annotations", {})
        if C.ANN_TRACE not in job.metadata["annotations"]:
            job.metadata["annotations"][C.ANN_TRACE] = json.dumps({"submitted": round(_t.time(), 4)})
        try:
            return self.jobs(ns).create(job)
        except APIError as e:
            if e.reason != "AlreadyExists":
                raise
            cur = self.jobs(ns).get(job.name)
            cur.spec = job.spec
            return self.jobs(ns).update(cur)

    def wait_for_phase(self, name: str, phases, namespace: str = "default", timeout: float = 60.0) -> AITrainingJob:
        if isinstance(phases, str):
            phases = (phases,)
        deadline = time.monotonic() + timeout
        job = None
        while time.monotonic() < deadline:
            try:
                job = self.jobs(namespace).get(name)
                if job.status.phase in phases:
                    return job
            except APIError:
                pass
            time.sleep(0.02)
        raise TimeoutError(f"job {name} did not reach {phases} within {timeout}s (phase={job.status.phase if job else None},"
                           f" conditions={[(c.type, c.message) for c in job.status.conditions] if job else None})")

    def pods(self, namespace: str = "default", selector: str = "") -> List[dict]:
        return self.clientset.core_v1().pods(namespace).list(selector).get("items", [])

    def stop(self, kill_workers: bool = True) -> None:
        self.stop_event.set()
        self.agent.shutdown(kill=kill_workers)
        for t in self._op_threads:
            t.join(timeout=3)
        if self.http:
            self.http.stop()

    def __enter__(self):
        return self.start()

    def __exit__(self, *exc):
        self.stop()


def _auto_pool(requested: int, gpus: Optional[int]) -> int:
    if requested >= 0:
        return requested
    from ..agent.agent import detect_gpu_count

    n = detect_gpu_count() if gpus is None else gpus
    return min(8, max(0, n))


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(prog="aitj-local", description="single-box AITrainingJob control plane")
    sub = ap.add_subparsers(dest="cmd", required=True)
    up = sub.add_parser("up", help="run API server + agent + operator(s) in the foreground")
    up.add_argument("--port", type=int, default=8001)
    up.add_argument("--gpus", type=int, default=None)
    up.add_argument("--workdir", default=os.path.expanduser("~/.aitj"))
    up.add_argument("--operators", type=int, default=1)
    up.add_argument("--leader-elect", action="store_true")
    up.add_argument("--no-wal", action="store_true")
    up.add_argument("--v", type=int, default=0)
    up.add_argument("--warm-pool", type=int, default=-1,
                    help="parked pre-imported interpreters for fast replica start (-1 = one per GPU slot, 0 = off)")
    up.add_argument("--gpu-visibility", default="pinned", choices=["pinned", "all"],
                    help="see aitj-agent --gpu-visibility")
    options_group = up.add_argument_group("operator flags")
    options_group.add_argument("--thread-num", type=int, default=4)
    options_group.add_argument("--enable-creating-failed", action="store_true")
    args = ap.parse_args(argv)
    opt = options_mod.TrainingJobOperatorOption(thread_num=args.thread_num,
                                                enable_creating_failed=args.enable_creating_failed, v=args.v)
    from ..signals import setup_signal_handler

    stop = setup_signal_handler()
    cluster = LocalCluster(num_gpus=args.gpus, workdir=args.workdir, wal=not args.no_wal, operators=args.operators,
                           leader_elect=args.leader_elect or args.operators > 1, port=args.port, option=opt,
                           verbosity=args.v, warm_pool=_auto_pool(args.warm_pool, args.gpus),
                           gpu_visibility=args.gpu_visibility)
    cluster.start()
    cfg_dir = os.path.expanduser("~/.aitj")
    os.makedirs(cfg_dir, exist_ok=True)
    with open(os.path.join(cfg_dir, "config"), "w") as f:
        f.write(f"server: {cluster.url}\n")
    print(f"aitj control plane up: {cluster.url}  (gpus={cluster.agent.num_gpus}, workdir={cluster.workdir})",
          flush=True)
    stop.wait()
    cluster.stop(kill_workers=False)
    return 0


if __name__ == "__main__":
    sys.exit(main())
