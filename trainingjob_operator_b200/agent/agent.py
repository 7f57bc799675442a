"""Node agent: the kube-scheduler + kubelet analogue for one 8xH100 box.

The reference has no such component -- it relies on Kubernetes to place pods, start containers and
report ``pod.status`` (SURVEY.md L0, Appendix A).  On a single box those roles collapse into this
agent, which keeps the exact object contract the controller logic reads
(/root/reference/pkg/controller/pod.go:339-379, status.go:339-358):

* **nodes**: one ``Node`` per GPU (``gpu-0`` .. ``gpu-7``, Ready <=> NVML health) plus ``cpu-0`` for
  replicas that request no GPU; "node not Ready" is how a GPU fault reaches the ``NodeFail`` path
  (pod.go:407-419).  Fault injection: annotate a node with ``aitj.b200/inject-fault``.
* **scheduler**: binds Pending pods (``spec.nodeName``) to free healthy GPUs, highest ``priority``
  label first (pod.go:503-505), honours ``schedulerName`` (pod.go:524-526) by ignoring pods addressed
  to a foreign scheduler; when nothing fits it writes the ``PodScheduled=False`` condition whose message
  the controller surfaces (pod.go:457-467).
* **kubelet**: one OS process (own process group) per container through the native supervisor
  (``core/csrc/supervisor.h``): ``CUDA_VISIBLE_DEVICES`` pinning, CPU affinity, log capture, init
  containers in order; ``containerStatuses`` waiting/running/terminated with exit codes (signal N =>
  128+N); exec failures surface as ``CreateContainerError`` / ``CreateContainerConfigError`` waiting
  reasons (constants.go:46-56); graceful delete = SIGTERM, grace period, SIGKILL, then the pod object
  is removed; a vanished pod object kills its processes (orphan sweep, garbage_collection.go analogue).
* **restart recovery**: ``containerStatuses[].containerID`` records ``aitj://<pid>/<start-time>``; a restarted agent
  re-adopts the workers of its predecessor that are still alive (identity = pid + kernel start time, exit observed
  through a pidfd) and fails the ones that are gone with ``ContainerStatusUnknown`` / 137, instead of leaving their
  pods ``Running`` forever or double-spawning them (SURVEY.md §7.3 item 4).  The exit status of an adopted (non-child)
  process cannot be waited for: a container that wrote its exit code to ``$AITJ_EXIT_FILE`` (the bundled workers do)
  is believed, any other is reported as ``ContainerStatusUnknown``.
* **liveness**: ``containers[].livenessProbe.exec`` is honoured (period / failureThreshold / initialDelay / timeout as
  in Kubernetes), and a worker that stops touching ``$AITJ_HEARTBEAT_FILE`` for ``AITJ_HANG_TIMEOUT`` seconds (env of
  the container) is treated the same way: event ``Unhealthy`` + ``Killing``, SIGKILL => exit 137 => the job's restart
  policy takes over.  This is the hang detection the reference leaves to kubelet probes (SURVEY.md §5.3); a DDP rank
  stuck in a collective because a peer died is the case it exists for.
(The scheduler, the liveness probes and the warm pool live in ``scheduler.py``, ``liveness.py`` and ``warmpool.py`` and are
mixed into ``NodeAgent``.)

* **warm pool** (``warm_pool=N``): N parked interpreters with torch already imported (``runtime/zygote.py``);
  a container whose command is ``python -m mod`` / ``python script`` adopts one instead of paying the
  interpreter start + ``import torch`` (seconds) on the spawn -> Running path (SURVEY.md §7.3 item 1).
"""
from __future__ import annotations

import os
import signal
import sys
import threading
import time
from dataclasses import dataclass, field
from typing import Any, Callable, Dict, List, Optional, Tuple

from ..api import constants as C
from ..api import meta as M
from ..client.informers import DeletedFinalStateUnknown, SharedInformerFactory
from ..client.record import EventRecorder
from ..core import _aitj_core as core
from ..store.apiserver import APIError
from ..utils import klog, lifecycle, metrics
from .liveness import LivenessMixin
from .scheduler import GPU_RESOURCE, OWN_SCHEDULERS, SchedulerMixin, pod_gpu_request, pod_priority  # noqa: F401
from .warmpool import PASS_ENV as _PASS_ENV
from .warmpool import ZYGOTE_PREFIX, WarmPoolMixin

metrics.describe("aitj_spawn_seconds", "pod bound -> all containers started")


def detect_gpu_count() -> int:
    env = os.environ.get("AITJ_NUM_GPUS")
    if env is not None:
        return int(env)
    try:
        import pynvml

        pynvml.nvmlInit()
        return int(pynvml.nvmlDeviceGetCount())
    except Exception:  # noqa: BLE001
        pass
    try:
        import torch

        return int(torch.cuda.device_count())
    except Exception:  # noqa: BLE001
        return 0


def nvml_health_prober() -> Callable[[int], Tuple[bool, str]]:
    """(healthy, reason) per GPU index from NVML; always healthy when NVML is unavailable."""
    try:
        import pynvml

        pynvml.nvmlInit()
    except Exception:  # noqa: BLE001
        return lambda idx: (True, "")

    def probe(idx: int) -> Tuple[bool, str]:
        try:
            h = pynvml.nvmlDeviceGetHandleByIndex(idx)
            pynvml.nvmlDeviceGetMemoryInfo(h)
            try:
                ecc = pynvml.nvmlDeviceGetTotalEccErrors(h, pynvml.NVML_MEMORY_ERROR_TYPE_UNCORRECTED,
                                                         pynvml.NVML_VOLATILE_ECC)
                if ecc and ecc > 0:
                    return False, f"{ecc} uncorrected volatile ECC errors"
            except Exception:  # noqa: BLE001 - not supported / disabled
                pass
            return True, ""
        except Exception as e:  # noqa: BLE001 - fallen off the bus, Xid, ...
            return False, f"NVML: {e}"

    return probe


def proc_start_time(pid: int) -> Optional[int]:
    """Kernel start time of ``pid`` in clock ticks since boot (field 22 of /proc/<pid>/stat) -- with the pid it
    identifies a process across agent restarts (pids are recycled, start times are not).  Read by the native core
    (no GIL hand-off per syscall on the container-start path)."""
    v = core.proc_start_time(int(pid))
    return int(v) if v else None


def container_id(pid: int) -> str:
    return f"aitj://{pid}/{proc_start_time(pid) or 0}"


def parse_container_id(cid: str) -> Tuple[int, int]:
    try:
        pid, start = cid[len("aitj://"):].split("/")
        return int(pid), int(start)
    except (ValueError, AttributeError):
        return 0, 0


class _RetryExit(Exception):
    """The API server could not be reached while a container exit was being recorded; the reaper tries again."""


@dataclass
class _PodState:
    key: str
    uid: str
    containers: Dict[str, str] = field(default_factory=dict)   # container name -> supervisor id
    started: bool = False
    running_unreported: bool = False      # containers are up but the Running status write did not reach the API server
    init_index: int = 0
    term_sent_at: float = 0.0
    bound_at: float = 0.0
    spawn_failures: int = 0
    next_retry: float = 0.0
    # serialises "containers started -> status Running" against the exit handler: a command that exits at once must not
    # have its terminated status overwritten by the (later) Running patch
    status_lock: threading.Lock = field(default_factory=threading.Lock)
    started_at: float = 0.0
    probe_next: Dict[str, float] = field(default_factory=dict)      # container -> next liveness check (monotonic)
    probe_failures: Dict[str, int] = field(default_factory=dict)


class NodeAgent(SchedulerMixin, WarmPoolMixin, LivenessMixin):
    def __init__(self, clientset, num_gpus: Optional[int] = None, workdir: str = "/tmp/aitj-agent",
                 health_prober: Optional[Callable[[int], Tuple[bool, str]]] = None, health_period: float = 2.0,
                 cpu_slots: int = 64, image_map: Optional[Dict[str, List[str]]] = None,
                 supervisor=None, node_prefix: str = "", warm_pool: int = 0, gpu_visibility: str = "pinned"):
        """``gpu_visibility``: how a replica is tied to its GPU slot.  ``pinned`` (default): ``CUDA_VISIBLE_DEVICES`` holds
        only the bound GPU(s) -- an opaque user container cannot touch anything else, which is what the reference's
        per-pod resource limits give it.  ``all``: every GPU of the box stays visible (natural order) and the bound one is
        named by ``LOCAL_RANK`` / ``AITJ_PINNED_GPU`` -- needed when the worker maps its peers' memory (CUDA symmetric
        memory refuses ranks that all call their device "0": the owner-sharded gradient path, ``parallel.symm``)."""
        self.gpu_visibility = gpu_visibility if gpu_visibility in ("pinned", "all") else "pinned"
        self.cs = clientset
        self.num_gpus = detect_gpu_count() if num_gpus is None else int(num_gpus)
        self.workdir = workdir
        self.log_dir = os.path.join(workdir, "logs")
        os.makedirs(self.log_dir, exist_ok=True)
        self.prober = health_prober or nvml_health_prober()
        self.health_period = health_period
        self.cpu_slots = cpu_slots
        self.image_map = image_map or {}
        self.sup = supervisor or core.Supervisor()
        self.prefix = node_prefix
        self.queue = core.WorkQueue("agent-pods", 0.02, 5.0, 200.0, 400)
        self._states: Dict[str, _PodState] = {}
        self._lock = threading.RLock()
        self._factory = SharedInformerFactory(clientset, 0.0)
        self._pod_informer = self._factory.core().v1().pods()
        self._node_informer = self._factory.core().v1().nodes()
        self._pod_informer.informer().add_event_handler(add=self._on_pod, update=lambda o, n: self._on_pod(n),
                                                        delete=self._on_pod_delete)
        self._node_informer.informer().add_event_handler(update=lambda o, n: self._kick_pending())
        self.pod_lister = self._pod_informer.lister()
        self.node_lister = self._node_informer.lister()
        self._threads: List[threading.Thread] = []
        self._injected: Dict[str, str] = {}
        self.recorder = EventRecorder(clientset, "aitj-agent", log=False)
        self.heartbeat_dir = os.path.join(workdir, "heartbeats")
        os.makedirs(self.heartbeat_dir, exist_ok=True)
        # authoritative GPU allocation table (gpu index -> pod uid): the informer cache lags behind our own
        # binds, so consecutive scheduling decisions must not rely on it alone
        self._gpu_owner: Dict[int, Tuple[str, float]] = {}
        self._bound: Dict[str, float] = {}   # pod uid -> time we bound it (cache may not show nodeName yet)
        self._unschedulable: set = set()     # keys of pods that did not fit; re-queued when a slot is released
        # warm pool of parked interpreters: supervisor id -> {"fifo": path, "spawned": monotonic}
        self.sync_workers = max(1, int(os.environ.get("AITJ_AGENT_SYNC_WORKERS", "1")))
        self.warm_pool = max(0, int(warm_pool))
        self._zygotes: Dict[str, Dict[str, Any]] = {}
        self._zy_seq = 0
        self._zy_failures = 0
        self._zy_dir = os.path.join(workdir, "zygotes")
        self._stopping = False

    # ------------------------------------------------------------------ nodes
    def gpu_node(self, idx: int) -> str:
        return f"{self.prefix}gpu-{idx}"

    @property
    def cpu_node(self) -> str:
        return f"{self.prefix}cpu-0"

    def node_names(self) -> List[str]:
        return [self.gpu_node(i) for i in range(self.num_gpus)] + [self.cpu_node]

    def register_nodes(self) -> None:
        for i in range(self.num_gpus):
            self._ensure_node(self.gpu_node(i), "gpu", {GPU_RESOURCE: "1"}, i)
        self._ensure_node(self.cpu_node, "cpu", {"cpu": str(os.cpu_count() or 1), "pods": str(self.cpu_slots)}, -1)

    def _ensure_node(self, name: str, ntype: str, capacity: Dict[str, str], gpu_index: int) -> None:
        node = {"apiVersion": "v1", "kind": "Node",
                "metadata": {"name": name, "labels": {"aitj.b200/type": ntype, "aitj.b200/gpu-index": str(gpu_index),
                                                      "kubernetes.io/hostname": name}},
                "spec": {},
                "status": {"capacity": capacity, "allocatable": capacity,
                           "conditions": [self._ready_condition(True, "KubeletReady", "agent is posting ready status")],
                           "nodeInfo": {"kubeletVersion": "aitj-agent/1.0", "architecture": "amd64"}}}
        try:
            self.cs.core_v1().nodes().create(node)
        except APIError as e:
            if e.reason != "AlreadyExists":
                raise
            self._set_node_ready(name, True, "KubeletReady", "agent is posting ready status")

    @staticmethod
    def _ready_condition(ok: bool, reason: str, message: str) -> dict:
        now = M.format_time()
        return {"type": "Ready", "status": "True" if ok else "False", "reason": reason, "message": message,
                "lastHeartbeatTime": now, "lastTransitionTime": now}

    def _set_node_ready(self, name: str, ok: bool, reason: str, message: str) -> None:
        try:
            node = self.cs.core_v1().nodes().get(name)
        except APIError:
            return
        conds = node.setdefault("status", {}).setdefault("conditions", [])
        cur = M.condition(conds, "Ready")
        want = "True" if ok else "False"
        if cur is not None and cur.get("status") == want and cur.get("reason") == reason:
            return
        new = self._ready_condition(ok, reason, message)
        if cur is None:
            conds.append(new)
        else:
            cur.update(new)
        try:
            self.cs.core_v1().nodes().update_status(node)
            klog.info("node %s Ready=%s (%s: %s)", name, want, reason, message)
        except APIError as e:
            klog.warning("node %s status update failed: %s", name, e.message)

    def _health_loop(self, stop: threading.Event) -> None:
        while not stop.wait(self.health_period):
            self.check_health_once()

    def check_health_once(self) -> None:
        for i in range(self.num_gpus):
            name = self.gpu_node(i)
            injected = ""
            try:
                node = self.node_lister.get(name)
                injected = M.annotations_of(node).get(C.ANN_INJECT_FAULT, "")
            except APIError:
                pass
            if injected:
                self._set_node_ready(name, False, "InjectedFault", injected)
                continue
            ok, why = self.prober(i)
            if ok:
                self._set_node_ready(name, True, "KubeletReady", "agent is posting ready status")
            else:
                self._set_node_ready(name, False, "GPUUnhealthy", why)

    # ------------------------------------------------------------------ informer handlers
    def _on_pod(self, pod: dict) -> None:
        self.queue.add(M.key_of(pod))

    def _on_pod_delete(self, obj) -> None:
        pod = obj.obj if isinstance(obj, DeletedFinalStateUnknown) else obj
        self.queue.add(M.key_of(pod))
        self._release_gpus(M.uid_of(pod))

    # ------------------------------------------------------------------ main loops
    def start(self, stop: threading.Event) -> None:
        self.register_nodes()
        self._factory.start(stop)
        self._factory.wait_for_cache_sync(stop)
        self.recover()
        # one sync worker by default: more (AITJ_AGENT_SYNC_WORKERS) are safe -- the queue hands a key to one worker at a
        # time and the scheduler's tables are guarded by self._lock -- but measured slower (GIL): 8-replica submit ->
        # Running p50 165 ms with one worker, 215 ms with four
        workers = [(self._sync_loop, f"agent-sync-{i}") for i in range(self.sync_workers)]
        for target, name in (*workers, (self._reap_loop, "agent-reap"),
                             (self._health_loop, "agent-health"), (self._sweep_loop, "agent-sweep"),
                             (self._probe_loop, "agent-liveness")):
            self._threads.append(lifecycle.spawn(target, name, (stop,)))
        lifecycle.register_stop(lambda: (stop.set(), self.queue.shutdown(), self._kill_zygotes()))
        threading.Thread(target=lambda: (stop.wait(), self.queue.shutdown(), self._kill_zygotes()),
                         daemon=True).start()
        self._ensure_pool()

    def recover(self) -> Dict[str, int]:
        """After an agent restart: re-adopt the still-running containers of pods bound to this agent's nodes and fail
        the ones whose process is gone.  Called from ``start`` before any pod is synced."""
        out = {"adopted": 0, "lost": 0}
        for pod in self.pod_lister.list():
            node = pod.get("spec", {}).get("nodeName") or ""
            status = pod.get("status", {})
            if not node or not self._mine(node) or status.get("phase") != C.POD_RUNNING:
                continue
            key = M.key_of(pod)
            with self._lock:
                if key in self._states:
                    continue
            st = _PodState(key=key, uid=M.uid_of(pod), bound_at=time.monotonic())
            st.started, st.started_at = True, time.monotonic()
            lost = []
            for cs in status.get("containerStatuses") or []:
                if "running" not in (cs.get("state") or {}):
                    continue
                pid, start = parse_container_id(cs.get("containerID", ""))
                sid = f"{key}/{st.uid[:8]}/{cs['name']}"
                if pid > 0 and start > 0 and proc_start_time(pid) == start:
                    try:
                        self.sup.adopt(sid, pid)
                        st.containers[cs["name"]] = sid
                        out["adopted"] += 1
                        continue
                    except OSError:
                        pass
                lost.append(cs["name"])
            gpus = [int(g) for g in (M.annotations_of(pod).get(C.ANN_GPUS) or "").split(",") if g.strip()]
            with self._lock:
                self._states[key] = st
                for g in gpus:
                    self._gpu_owner[g] = (st.uid, time.monotonic())
            if lost:
                out["lost"] += len(lost)
                now = M.format_time()
                statuses = M.deepcopy(status.get("containerStatuses") or [])
                for cs in statuses:
                    if cs.get("name") in lost:
                        cs["ready"] = False
                        cs["state"] = {"terminated": {"exitCode": 137, "reason": "ContainerStatusUnknown", "finishedAt": now,
                                                      "message": "process lost across an agent restart"}}
                self._kill_pod_processes(key, signal.SIGKILL)      # a pod is all-or-nothing: stop its other containers
                try:
                    self.cs.core_v1().pods(M.namespace_of(pod)).patch(
                        M.name_of(pod), {"status": {"phase": C.POD_FAILED, "containerStatuses": statuses}},
                        subresource="status")
                except APIError as e:
                    klog.warning("recover: status update of %s failed: %s", key, e.message)
                self._release_gpus(st.uid)
        if out["adopted"] or out["lost"]:
            klog.info("agent restart recovery: adopted %d running container(s), %d lost", out["adopted"], out["lost"])
        return out

    def run(self, stop: threading.Event) -> None:
        self.start(stop)
        stop.wait()
        self.shutdown()

    def shutdown(self, kill: bool = False) -> None:
        self._kill_zygotes()
        if kill:
            for sid, _pid in self.sup.list():
                self.sup.kill(sid, signal.SIGKILL, True)

    def _sync_loop(self, stop: threading.Event) -> None:
        while not stop.is_set():
            key = self.queue.get(0.5)
            if key is None:
                if self.queue.shutting_down():
                    return
                continue
            try:
                self.sync_pod(key)
                self.queue.forget(key)
            except APIError as e:
                if e.reason not in ("NotFound",):
                    klog.V(2).info("agent: sync %s: %s", key, e.message)
                    self.queue.add_rate_limited(key)
            except Exception as e:  # noqa: BLE001
                klog.error("agent: sync %s failed: %r", key, e)
                self.queue.add_rate_limited(key)
            finally:
                self.queue.done(key)

    def _reap_loop(self, stop: threading.Event) -> None:
        retry: List[Dict[str, Any]] = []       # exits whose status write did not reach the API server yet
        while not stop.is_set():
            events = self.sup.poll_exits(0.5)
            again, retry = retry, []
            for ev in again + list(events):
                if ev["id"].startswith(ZYGOTE_PREFIX):
                    self._on_zygote_exit(ev)
                    continue
                try:
                    self._on_exit(ev)
                except _RetryExit as e:
                    # kubelet semantics: a container's termination is reported until the API server has it -- an exit that
                    # happens while the server is restarting must not leave the pod Running forever
                    klog.V(2).info("agent: exit of %s not recorded yet (%s), will retry", ev["id"], e)
                    retry.append(ev)

    def _sweep_loop(self, stop: threading.Event) -> None:
        n = 0
        while not stop.wait(5.0):
            self.sweep_orphans()
            n += 1
            if n % 120 == 0:                  # every ten minutes
                self.sweep_files()

    def sweep_files(self, retention_s: Optional[float] = None) -> int:
        """Container logs, heartbeat and exit-code files outlive their pod on purpose (``aitjctl logs`` of a finished
        replica, post-mortems; kubelet would delete them with the pod) -- but not forever: files of pods that no longer
        exist are removed once they have not been written for ``AITJ_LOG_RETENTION`` seconds (default one day)."""
        if retention_s is None:
            retention_s = float(os.environ.get("AITJ_LOG_RETENTION", "86400"))
        live = {f"{M.namespace_of(p)}_{M.name_of(p)}_" for p in self.pod_lister.peek()}
        now, removed = time.time(), 0
        for d in (self.log_dir, self.heartbeat_dir):
            try:
                names = os.listdir(d)
            except OSError:
                continue
            for fn in names:
                if any(fn.startswith(prefix) for prefix in live):
                    continue
                path = os.path.join(d, fn)
                try:
                    if now - os.stat(path).st_mtime > retention_s:
                        os.unlink(path)
                        removed += 1
                except OSError:
                    pass
        return removed

    # ------------------------------------------------------------------ per-pod sync
    def _mine(self, node_name: str) -> bool:
        return node_name in self.node_names()

    def sync_pod(self, key: str) -> None:
        ns, name = M.split_key(key)
        try:
            pod = self.pod_lister.namespaced(ns).get(name)
        except APIError:
            self._kill_pod_processes(key, signal.SIGKILL)
            with self._lock:
                gone = self._states.pop(key, None)
            if gone is not None:
                self._release_gpus(gone.uid)
            return
        st = self._states.get(key)
        if st is not None and st.uid != M.uid_of(pod):
            # same name, new incarnation: the old processes must not survive
            self._kill_pod_processes(key, signal.SIGKILL)
            with self._lock:
                self._states.pop(key, None)
            st = None
        node = pod.get("spec", {}).get("nodeName") or ""
        if pod.get("metadata", {}).get("deletionTimestamp"):
            if not node or self._mine(node):
                self._terminate(pod, key)
            return
        phase = pod.get("status", {}).get("phase") or C.POD_PENDING
        if not node:
            if phase == C.POD_PENDING and not (st is not None and st.started):
                self.schedule(pod)          # (started: the cache is behind a bind + direct start of this very pod)
            return
        if not self._mine(node):
            return
        if phase == C.POD_PENDING:
            self._start_pod(pod, key)

    # ------------------------------------------------------------------ kubelet: start
    def _container_argv(self, c: dict) -> Tuple[Optional[List[str]], str]:
        cmd = list(c.get("command") or [])
        args = list(c.get("args") or [])
        if not cmd:
            mapped = self.image_map.get(c.get("image", ""))
            if mapped:
                cmd = list(mapped)
            elif not args:
                return None, (f"container {c.get('name')}: no command; image {c.get('image')!r} cannot be pulled on a "
                              "single box (pass --image-map image=command)")
        return [str(x) for x in cmd + args], ""

    def _container_env(self, pod: dict, c: dict, gpus: List[int]) -> Dict[str, str]:
        env = {k: os.environ[k] for k in _PASS_ENV if k in os.environ}
        share = self.gpu_visibility == "all" and len(gpus) == 1 and self.num_gpus > 1
        env["CUDA_VISIBLE_DEVICES"] = ",".join(str(g) for g in (range(self.num_gpus) if share else gpus))
        env["CUDA_DEVICE_ORDER"] = "PCI_BUS_ID"
        env["AITJ_PINNED_GPU"] = ",".join(str(g) for g in gpus)
        env.setdefault("NCCL_IB_DISABLE", "1")
        env.setdefault("NCCL_SOCKET_IFNAME", "lo")
        env["AITJ_POD_NAME"] = M.name_of(pod)
        env["AITJ_POD_NAMESPACE"] = M.namespace_of(pod)
        env["AITJ_POD_UID"] = M.uid_of(pod)
        env["AITJ_NODE_NAME"] = pod.get("spec", {}).get("nodeName", "")
        env["AITJ_WORKDIR"] = self.workdir
        env["AITJ_HEARTBEAT_FILE"] = self.heartbeat_path(pod, c.get("name", ""))
        env["AITJ_EXIT_FILE"] = self.heartbeat_path(pod, c.get("name", "")) + ".exit"
        env["PYTHONUNBUFFERED"] = "1"
        for e in c.get("env") or []:
            if "name" in e:
                env[str(e["name"])] = str(e.get("value", ""))
        if share:
            env["LOCAL_RANK"] = str(gpus[0])       # the bound GPU, among all the visible ones
        return env

    def _cpus_for(self, gpus: List[int]) -> List[int]:
        ncpu = os.cpu_count() or 1
        if not gpus or self.num_gpus <= 0 or ncpu < self.num_gpus * 2:
            return []
        per = ncpu // self.num_gpus
        out: List[int] = []
        for g in gpus:
            out += list(range(g * per, (g + 1) * per))
        return out

    def heartbeat_path(self, pod: dict, container: str) -> str:
        return os.path.join(self.heartbeat_dir, f"{M.namespace_of(pod)}_{M.name_of(pod)}_{container}")

    def log_path(self, pod: dict, container: str) -> str:
        return os.path.join(self.log_dir, f"{M.namespace_of(pod)}_{M.name_of(pod)}_{container}.log")

    def _start_pod(self, pod: dict, key: str) -> None:
        with self._lock:
            st = self._states.get(key)
            if st is None:
                st = self._states[key] = _PodState(key=key, uid=M.uid_of(pod), bound_at=time.monotonic())
            if (st.started and not st.running_unreported) or time.monotonic() < st.next_retry:
                return
        with st.status_lock:
            self._start_pod_locked(pod, st)

    def _start_pod_locked(self, pod: dict, st: _PodState) -> None:
        spec = pod.get("spec", {})
        gpus = [int(g) for g in (M.annotations_of(pod).get(C.ANN_GPUS) or "").split(",") if g.strip()]
        inits = spec.get("initContainers") or []
        mains = spec.get("containers") or []
        # init containers run one at a time; `_on_exit` advances the index
        if st.init_index < len(inits):
            c = inits[st.init_index]
            if c["name"] not in st.containers:
                self._spawn_container(pod, st, c, gpus, init=True)
            return
        statuses = []
        ok = True
        if st.started and st.running_unreported and not all(
                self.sup.alive(st.containers.get(c["name"], "")) for c in mains):
            st.running_unreported = False      # a container has exited meanwhile: the exit path reports from here on
            return
        for c in mains:
            if c["name"] in st.containers:
                continue
            err = self._spawn_container(pod, st, c, gpus, init=False)
            if err:
                ok = False
                break
        if not ok:
            return
        st.started = True
        st.started_at = time.monotonic()
        now = M.format_time()
        for c in mains:
            statuses.append({"name": c["name"], "image": c.get("image", ""), "ready": True, "restartCount": 0,
                             "containerID": container_id(self.sup.pid_of(st.containers[c["name"]])),
                             "state": {"running": {"startedAt": now}}})
        patch = {"status": {"phase": C.POD_RUNNING, "startTime": pod.get("status", {}).get("startTime") or now,
                            "containerStatuses": statuses,
                            "conditions": [{"type": "PodScheduled", "status": "True"},
                                           {"type": "Ready", "status": "True", "lastTransitionTime": now}]}}
        try:
            self.cs.core_v1().pods(M.namespace_of(pod)).patch(M.name_of(pod), patch, subresource="status")
        except APIError:
            st.running_unreported = True       # the sync loop re-queues the pod; only the status write is repeated
            raise
        st.running_unreported = False
        metrics.observe("aitj_spawn_seconds", time.monotonic() - st.bound_at)

    def _spawn_container(self, pod: dict, st: _PodState, c: dict, gpus: List[int], init: bool) -> str:
        argv, err = self._container_argv(c)
        reason = "CreateContainerConfigError"
        if argv is not None:
            sid = f"{st.key}/{st.uid[:8]}/{c['name']}"
            try:
                cwd = c.get("workingDir") or ""
                env = self._container_env(pod, c, gpus)
                log, cpus = self.log_path(pod, c["name"]), self._cpus_for(gpus)
                if "AITJ_HANG_TIMEOUT" in env:
                    try:    # a fresh heartbeat: a restarted replica must not inherit its predecessor's stale one
                        with open(env["AITJ_HEARTBEAT_FILE"], "w"):
                            pass
                    except OSError:
                        pass
                try:
                    os.unlink(env["AITJ_EXIT_FILE"])
                except OSError:
                    pass
                if not self._adopt_zygote(sid, argv, env, cwd, log, cpus):
                    self.sup.spawn(sid, argv, env, cwd, log, "", cpus)
                st.containers[c["name"]] = sid
                return ""
            except OSError as e:
                err = str(e)
                reason = "CreateContainerError"
        st.spawn_failures += 1
        st.next_retry = time.monotonic() + min(30.0, 0.5 * (2 ** min(st.spawn_failures, 6)))
        self.queue.add_after(st.key, st.next_retry - time.monotonic() + 0.01)
        now = M.format_time()
        cs = {"name": c["name"], "image": c.get("image", ""), "ready": False, "restartCount": 0,
              "state": {"waiting": {"reason": reason, "message": err}}}
        patch = {"status": {"phase": C.POD_PENDING, "startTime": pod.get("status", {}).get("startTime") or now,
                            "containerStatuses": [cs]}}
        try:
            self.cs.core_v1().pods(M.namespace_of(pod)).patch(M.name_of(pod), patch, subresource="status")
        except APIError:
            pass
        klog.warning("pod %s container %s: %s: %s", st.key, c["name"], reason, err)
        return err or reason

    # ------------------------------------------------------------------ kubelet: exits
    def _on_exit(self, ev: Dict[str, Any]) -> None:
        sid = ev["id"]
        key = "/".join(sid.split("/")[:2])
        cname = sid.split("/")[-1]
        with self._lock:
            st = self._states.get(key)
        if st is None:
            return
        with st.status_lock:      # the start path holds it across spawn + bookkeeping: a process that exits at once
            if st.containers.get(cname) != sid:          # is only looked up after its id has been recorded
                return
            self._on_exit_locked(ev, st, key, cname)

    def _on_exit_locked(self, ev: Dict[str, Any], st: _PodState, key: str, cname: str) -> None:
        ns, name = M.split_key(key)
        try:
            pod = self.cs.core_v1().pods(ns).get(name)
        except APIError as e:
            if e.reason == "NotFound":
                return
            raise _RetryExit(e.message) from None
        if M.uid_of(pod) != st.uid:
            return
        code, sig = int(ev["exit_code"]), int(ev["signal"])
        now = M.format_time()
        if ev.get("status_unknown"):
            # adopted after an agent restart: not our child, so no wait status.  A container that recorded its own exit
            # code in $AITJ_EXIT_FILE (our workers do; any command may) is believed, anything else is "unknown" = 137
            recorded = None
            try:
                with open(self.heartbeat_path(pod, cname) + ".exit") as f:
                    recorded = int(f.read().strip() or "x")
            except (OSError, ValueError):
                pass
            if recorded is not None:
                code, sig = recorded, 0
                ev = dict(ev, status_unknown=False)
        term = {"exitCode": code, "reason": "Completed" if code == 0 else "Error", "finishedAt": now}
        if ev.get("status_unknown"):
            term["reason"] = "ContainerStatusUnknown"
            term["message"] = "the container was adopted after an agent restart; its exit status could not be read"
        if sig:
            term["signal"] = sig
            term["message"] = f"killed by signal {sig}"
        inits = [c["name"] for c in pod.get("spec", {}).get("initContainers") or []]
        if cname in inits:
            if code == 0:
                st.init_index += 1
                st.containers.pop(cname, None)
                self.queue.add(key)
                return
            patch = {"status": {"phase": C.POD_FAILED, "reason": "InitContainerFailed",
                                "message": f"init container {cname} exited with {code}",
                                "initContainerStatuses": [{"name": cname, "state": {"terminated": term}}]}}
            try:
                self.cs.core_v1().pods(ns).patch(name, patch, subresource="status")
            except APIError as e:
                if e.reason != "NotFound":
                    raise _RetryExit(e.message) from None
            return
        statuses = M.deepcopy(pod.get("status", {}).get("containerStatuses") or [])
        found = False
        for cs in statuses:
            if cs.get("name") == cname:
                cs["state"] = {"terminated": term}
                cs["ready"] = False
                found = True
        if not found:
            statuses.append({"name": cname, "ready": False, "restartCount": 0, "state": {"terminated": term}})
        want = [c["name"] for c in pod.get("spec", {}).get("containers") or []]
        terms = {cs["name"]: cs["state"]["terminated"] for cs in statuses if "terminated" in (cs.get("state") or {})}
        status: Dict[str, Any] = {"containerStatuses": statuses}
        if all(n in terms for n in want):
            status["phase"] = C.POD_SUCCEEDED if all(terms[n]["exitCode"] == 0 for n in want) else C.POD_FAILED
        if "phase" in status:
            self._release_gpus(st.uid, kick=False)      # pending pods are kicked below, after the status write
        klog.V(2).info("pod %s container %s exited code=%d signal=%d", key, cname, code, sig)
        try:
            self.cs.core_v1().pods(ns).patch(name, {"status": status}, subresource="status")
        except APIError as e:
            if e.reason != "NotFound":
                raise _RetryExit(e.message) from None
        self._kick_pending()

    # ------------------------------------------------------------------ kubelet: terminate
    def _alive_ids(self, key: str) -> List[str]:
        with self._lock:
            st = self._states.get(key)
            ids = list(st.containers.values()) if st else []
        return [sid for sid in ids if self.sup.alive(sid)]

    def _kill_pod_processes(self, key: str, sig: int) -> None:
        for sid in self._alive_ids(key):
            self.sup.kill(sid, sig, True)

    def _terminate(self, pod: dict, key: str) -> None:
        alive = self._alive_ids(key)
        ns, name = M.namespace_of(pod), M.name_of(pod)
        if not alive:
            try:
                self.cs.core_v1().pods(ns).delete(name, grace_period_seconds=0)
            except APIError as e:
                if e.reason != "NotFound":
                    raise
            with self._lock:
                self._states.pop(key, None)
            self._kick_pending()
            return
        grace = float(pod["metadata"].get("deletionGracePeriodSeconds") or 0)
        age = M.seconds_since(pod["metadata"].get("deletionTimestamp"))
        with self._lock:
            st = self._states.get(key)
        if st is not None and not st.term_sent_at:
            st.term_sent_at = time.monotonic()
            self._kill_pod_processes(key, signal.SIGTERM)
        if age >= grace or (st is not None and time.monotonic() - st.term_sent_at >= grace):
            self._kill_pod_processes(key, signal.SIGKILL)
        self.queue.add_after(key, 0.05 if grace <= 1 else 0.2)

    # ------------------------------------------------------------------ orphan sweep
    def sweep_orphans(self) -> int:
        """Kill supervised processes whose pod record is gone or was replaced (GC analogue)."""
        n = 0
        for sid, _pid in self.sup.list():
            if sid.startswith(ZYGOTE_PREFIX):
                continue
            key = "/".join(sid.split("/")[:2])
            uid8 = sid.split("/")[2] if sid.count("/") >= 3 else ""
            ns, name = M.split_key(key)
            try:
                pod = self.pod_lister.namespaced(ns).get(name)
                if not uid8 or M.uid_of(pod).startswith(uid8):
                    continue
            except APIError:
                pass
            klog.info("orphan process %s: owning pod is gone, killing", sid)
            self.sup.kill(sid, signal.SIGKILL, True)
            n += 1
        return n
