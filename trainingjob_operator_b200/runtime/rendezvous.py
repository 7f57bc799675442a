"""Process-group membership of a worker: bounded, interruptible rendezvous on the job's current generation, the elected
state hand-off after every (re-)rendezvous, and what a ``faultTolerant`` job needs when a peer dies under a collective
(drop / abort the broken group, wait for the controller's next generation, the NCCL stall breaker).  The heartbeat the
node agent's hang detection reads lives here too, because every legitimately blocking wait in this module keeps it going.

The reference has none of this: it starts N containers with a fixed environment and never tells them anything again
(/root/reference/pkg/controller/pod.go:528, SURVEY.md §2.4 "Elastic DP", §5.3).
"""
from __future__ import annotations

import contextlib
import gc
import os
import threading
import time
from typing import Any, Dict, Optional

import torch
import torch.distributed as dist

_HB = {"path": os.environ.get("AITJ_HEARTBEAT_FILE", ""), "last": 0.0}


def heartbeat(force: bool = False) -> None:
    """Touch ``$AITJ_HEARTBEAT_FILE`` (at most once a second): the node agent kills a worker whose heartbeat is older
    than the container's ``AITJ_HANG_TIMEOUT`` -- e.g. a rank stuck in a collective after a peer died."""
    path = _HB["path"] or os.environ.get("AITJ_HEARTBEAT_FILE", "")
    now = time.time()
    if not path or (not force and now - _HB["last"] < 1.0):
        return
    _HB["last"] = now
    try:
        with open(path, "a"):
            os.utime(path, None)
    except OSError:
        pass


class StaleGeneration(RuntimeError):
    """The job moved on to a newer rendezvous generation while this rank was waiting for its peers."""


def init_process_group(rank: int, world: int, port: int, device: torch.device, timeout_s: float = 120.0,
                       attempt_timeout_s: float = 0.0, stale=None):
    """Rendezvous on the generation's loopback port.  With ``attempt_timeout_s`` the gathering phase (all ranks
    present) is bounded separately and raises on expiry, so the caller can re-read the job's current rendezvous
    generation and try again; ``timeout_s`` stays the collective timeout of the process group.  ``stale()`` is polled
    while gathering: when it turns true (the controller published a newer generation) the wait ends at once with
    ``StaleGeneration`` instead of sitting out the attempt."""
    import datetime

    backend = "nccl" if device.type == "cuda" else "gloo"
    kw: Dict[str, Any] = {}
    if device.type == "cuda":
        kw["device_id"] = device
    if attempt_timeout_s > 0:
        deadline = time.time() + attempt_timeout_s
        if rank != 0:
            # TCPStore's own connect loop backs off exponentially (tens of seconds once the master is half a minute
            # late, e.g. a replacement rank 0 that is still importing torch): probe the port ourselves at a fixed 50 ms
            _wait_for_listener(port, attempt_timeout_s, stale)
        # the store does not wait for the workers itself (that wait cannot be interrupted): every rank files a key and
        # polls for the others', so the gathering is bounded by *our* deadline and ends early on a newer generation
        store = dist.TCPStore("127.0.0.1", port, world, is_master=(rank == 0),
                              timeout=datetime.timedelta(seconds=max(1.0, deadline - time.time())),
                              wait_for_workers=False)
        try:
            _gather_ranks(store, rank, world, deadline, stale)
            store.set_timeout(datetime.timedelta(seconds=timeout_s))
            dist.init_process_group(backend, store=store, rank=rank, world_size=world,
                                    timeout=datetime.timedelta(seconds=timeout_s), **kw)
        except BaseException:
            if dist.is_initialized():
                dist.destroy_process_group()
            del store                     # closes the listening socket: the next attempt may use the same port
            gc.collect()
            raise
        return
    dist.init_process_group(backend, init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world,
                            timeout=datetime.timedelta(seconds=timeout_s), **kw)


def _gather_ranks(store, rank: int, world: int, deadline: float, stale) -> None:
    keys = [f"aitj/arrived/{r}" for r in range(world)]
    store.set(keys[rank], "1")            # idempotent: a rank that retries on the same store does not count twice
    next_stale_check = 0.0
    while not store.check(keys):
        now = time.time()
        if now > deadline:
            raise TimeoutError(f"only some of the {world} ranks arrived on the rendezvous store")
        if stale is not None and now >= next_stale_check:
            next_stale_check = now + 0.25
            if stale():
                raise StaleGeneration("a newer rendezvous generation was published")
        time.sleep(0.01)


def _wait_for_listener(port: int, timeout_s: float, stale=None) -> bool:
    import socket

    deadline = time.time() + timeout_s
    next_stale_check = time.time() + 0.25
    while time.time() < deadline:
        try:
            socket.create_connection(("127.0.0.1", port), timeout=1.0).close()
            return True
        except OSError:
            time.sleep(0.05)
        if stale is not None and time.time() >= next_stale_check:
            next_stale_check = time.time() + 0.25
            if stale():
                raise StaleGeneration("a newer rendezvous generation was published")
    return False


class _KeepBeating:
    """Heart-beats from a side thread while the main thread is legitimately blocked in a *bounded* wait (waiting for
    peers in a rendezvous attempt); a stuck training step still stops the heartbeat, which is the point of it."""

    def __enter__(self):
        self._stop = threading.Event()
        self._t = threading.Thread(target=self._run, daemon=True)
        self._t.start()
        return self

    def _run(self):
        while not self._stop.wait(1.0):
            heartbeat(force=True)

    def __exit__(self, *exc):
        self._stop.set()
        self._t.join(timeout=2.0)
        return False


def rendezvous(rank: int, rdv: Dict[str, int], device: torch.device, watcher) -> Optional[Dict[str, int]]:
    """Join the job's CURRENT rendezvous generation.  A replica created for generation g may find, while it waits for
    its peers, that the controller has moved on (another replica failed and was re-created, the job was rescaled): the
    attempt is bounded (``AITJ_RDV_ATTEMPT_TIMEOUT``, default 30 s), after which the newest generation / world / port
    is read from the job and the rendezvous is retried there, so replicas created at different moments converge
    instead of waiting for each other on different ports.  Returns the adopted record, or None when this rank is no
    longer part of the world."""
    attempt = float(os.environ.get("AITJ_RDV_ATTEMPT_TIMEOUT", "30"))
    deadline = time.time() + float(os.environ.get("AITJ_RDV_TIMEOUT", "600"))
    # Collective timeout of the group.  gloo does not always fail a receive that is posted on a connection its peer's
    # death already closed -- the rank then sits out the whole timeout before the faultTolerant recovery can start, and
    # a blocked gloo collective cannot be aborted from another thread (NCCL can: StallBreaker) -- so a faultTolerant
    # CPU job gets a short one.
    coll_timeout = float(os.environ.get("AITJ_COLLECTIVE_TIMEOUT", "0")) or \
        (15.0 if device.type == "cpu" and os.environ.get("AITJ_FAULT_TOLERANT") == "1" else 120.0)
    cur = dict(rdv)
    while True:
        latest = watcher.fetch_now() if watcher is not None else None
        if latest is not None and latest["generation"] > cur["generation"]:
            print(f"[worker {rank}] rendezvous: generation {cur['generation']} is stale, joining {latest['generation']} "
                  f"(world {latest['world']})", flush=True)
            cur = {"generation": latest["generation"], "world": latest["world"], "port": latest["port"]}
        if rank >= cur["world"]:
            return None
        if cur["world"] <= 1:
            return cur
        try:
            with _KeepBeating():
                gen_now = cur["generation"]

                def stale() -> bool:
                    r = watcher.fetch_now()
                    return r is not None and r["generation"] > gen_now

                init_process_group(rank, cur["world"], cur["port"], device, timeout_s=coll_timeout,
                                   attempt_timeout_s=attempt if watcher is not None else 0.0,
                                   stale=stale if watcher is not None else None)
            return cur
        except Exception as e:  # noqa: BLE001 - peers missing within the attempt window (or a stale port)
            if dist.is_initialized():
                dist.destroy_process_group()
            if watcher is None or time.time() > deadline:
                raise
            print(f"[worker {rank}] rendezvous attempt on generation {cur['generation']} failed "
                  f"({type(e).__name__}); re-reading the job", flush=True)
            heartbeat(force=True)


def max_over_ranks(value: float, device: torch.device) -> float:
    if not dist.is_initialized() or dist.get_world_size() == 1:
        return value
    t = torch.tensor([value], dtype=torch.float64, device=device if device.type == "cuda" else "cpu")
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t[0])


def sync_state(adapter, loop_step: int, device: torch.device, have_state: bool = True) -> int:
    """Hand-off after every (re-)rendezvous.  The source is elected, not assumed to be rank 0: the rank holding the most
    optimizer steps wins (ties: the lowest rank; ranks that only have a throw-away warm-up state bid -1), so when rank 0
    itself was the replica that got replaced, its replacement receives the survivors' state instead of overwriting it.
    The source broadcasts {optimizer step, loop step, data position} and then the flat state tensors.  Same call sequence
    on every rank.  The data position (samples of a token corpus the job has consumed) is taken from adapters that keep
    one and given to them; others send 0."""
    if not dist.is_initialized() or dist.get_world_size() <= 1:
        return loop_step
    from ..parallel.ddp import broadcast_state

    world, rank = dist.get_world_size(), dist.get_rank()
    cdev = device if device.type == "cuda" else "cpu"
    bid = torch.tensor([int(adapter.step_count) * world + (world - 1 - rank) if have_state else -1],
                       dtype=torch.int64, device=cdev)
    dist.all_reduce(bid, op=dist.ReduceOp.MAX)
    best = int(bid[0])
    src = 0 if best < 0 else world - 1 - (best % world)
    st = torch.tensor([adapter.step_count, loop_step, int(getattr(adapter, "data_position", 0))], dtype=torch.int64,
                      device=cdev)
    dist.broadcast(st, src)
    broadcast_state(adapter.state_tensors(), src)
    adapter.after_state_load()
    adapter.step_count = int(st[0])
    if hasattr(adapter, "data_position"):
        adapter.data_position = int(st[2])
    return int(st[1])


# ------------------------------------------------------------------------------------ fault tolerance
def teardown_group(broken: bool = False) -> None:
    """Leave the current process group.  A group with a dead peer is *aborted* (NCCL: ``ncclCommAbort`` unblocks kernels
    that wait for the peer; a clean destroy would wait for them), a healthy one is destroyed."""
    if not dist.is_initialized():
        return
    if broken and dist.get_backend() == "nccl":
        try:
            from torch.distributed.distributed_c10d import _abort_process_group

            _abort_process_group()
            return
        except Exception as e:  # noqa: BLE001
            print(f"[worker] abort of the process group failed ({type(e).__name__}: {e}); destroying it", flush=True)
    try:
        dist.destroy_process_group()
    except Exception as e:  # noqa: BLE001 - sockets of a dead peer
        print(f"[worker] destroy of the broken process group raised {type(e).__name__}", flush=True)


def wait_for_newer_generation(watcher, generation: int, timeout_s: float, should_stop=None) -> Optional[Dict[str, int]]:
    """After a peer was lost: the controller replaces it and publishes the next rendezvous generation; poll for it.
    ``should_stop()`` (SIGTERM received: the job is being torn down instead of repaired) ends the wait."""
    deadline = time.time() + timeout_s
    while time.time() < deadline and not (should_stop is not None and should_stop()):
        latest = watcher.fetch_now()
        if latest is not None and latest["generation"] > generation:
            return latest
        heartbeat(force=True)
        time.sleep(0.05)
    return None


class StallBreaker:
    """NCCL has no error to raise when a peer dies: the surviving ranks' kernels spin on the dead peer's flags until the
    watchdog gives up (minutes) and takes the process down.  For a ``faultTolerant`` job this side thread aborts the
    communicator instead, once (a) the controller has published a newer rendezvous generation (= it replaced a replica)
    and (b) the main thread has not reached a step boundary for ``after_s`` seconds; the blocked step then fails and the
    main thread takes the same recovery path as an exception from gloo.  Only armed on CUDA (``AITJ_FT_ABORT_AFTER``,
    default 3 s, 0 disables)."""

    def __init__(self, watcher, after_s: float, action: str = "abort"):
        """``action="abort"``: abort the communicator (faultTolerant jobs recover in place).  ``action="exit"``: this
        replica cannot recover in place (owner-sharded state, no faultTolerant flag) -- it leaves with exit code 137 right
        away, as the agent's hang detection would after ``AITJ_HANG_TIMEOUT``, so that a ``restartScope: Pod`` job whose
        survivors sit in a dead collective is whole again in seconds instead of after the heartbeat time-out."""
        self.watcher, self.after_s, self.action = watcher, after_s, action
        self.generation = 0
        self.last_progress = time.time()
        self.in_step = False          # only a rank that sits inside a training step can be stuck behind a dead peer
        # how long one step may take before it counts as stuck: ``after_s``, except for the first step after a (re-)bind,
        # which legitimately takes seconds (kernel loading, CUDA-graph capture) -- the worker raises it for that step
        self.patience = after_s
        self._measured_generation = None    # generation whose steps the patience follows (begin_step / step_done)
        self._first_step = 0.0
        self._slowest_steady: Optional[float] = None
        self.tripped = False
        self._stop = threading.Event()
        self._t = threading.Thread(target=self._run, name="stall-breaker", daemon=True)
        self._t.start()

    FIRST_STEP_S = 30.0     # patience for the first step on a freshly bound trainer (kernel loading, graph capture)

    def begin_step(self, generation: int) -> None:
        """At a step boundary: the patience for the coming step, from the steps this generation has completed.  None yet:
        ``FIRST_STEP_S``.  Only the first: twice that step -- it did everything a steady step does and also loaded
        kernels and captured graphs, so it bounds a steady step from above.  Otherwise twice the slowest steady step -- a
        step that accumulates many micro-batches legitimately takes seconds.  Never less than ``after_s``."""
        if self._measured_generation != generation:
            self.patience = max(self.after_s, self.FIRST_STEP_S)
        elif self._slowest_steady is None:
            self.patience = max(self.after_s, 2.0 * self._first_step)
        else:
            self.patience = max(self.after_s, 2.0 * self._slowest_steady)

    def step_done(self, generation: int, seconds: float) -> None:
        """A training step of ``generation`` completed in ``seconds``."""
        if self._measured_generation != generation:
            self._measured_generation, self._first_step, self._slowest_steady = generation, seconds, None
        else:
            self._slowest_steady = max(self._slowest_steady or 0.0, seconds)

    def progress(self, generation: int) -> None:
        self.generation = generation
        self.last_progress = time.time()

    def _run(self) -> None:
        while not self._stop.wait(0.5):
            if self.tripped or not self.in_step or time.time() - self.last_progress < self.patience \
                    or not dist.is_initialized():
                continue
            latest = self.watcher.fetch_now()
            if latest is None or latest["generation"] <= self.generation:
                continue
            if self.action == "exit":
                print(f"[worker] no step boundary for {time.time() - self.last_progress:.1f}s while generation "
                      f"{latest['generation']} is pending: a peer is gone and this job does not recover in place -- "
                      f"leaving (137) so the controller replaces this replica too", flush=True)
                path = os.environ.get("AITJ_EXIT_FILE", "")
                if path:
                    try:
                        with open(path, "w") as f:
                            f.write("137")
                    except OSError:
                        pass
                os._exit(137)
            print(f"[worker] no step boundary for {time.time() - self.last_progress:.1f}s while generation "
                  f"{latest['generation']} is pending: aborting the communicator", flush=True)
            self.tripped = True
            teardown_group(broken=True)

    def stop(self) -> None:
        self._stop.set()


@contextlib.contextmanager
def guarded(breaker, what: str, generation: Optional[int] = None):
    """Run the body as "inside a step" for ``breaker`` (a StallBreaker; None: the body runs as is): a collective in it
    that hangs behind a dead peer gets the communicator aborted, and the abort surfaces here as a RuntimeError naming
    ``what``, which the training loop's recovery path handles.  ``generation``: the body starts at a step boundary of it
    -- only a newer generation (another peer lost meanwhile) makes the breaker abort."""
    if breaker is None:
        yield
        return
    if generation is not None:
        breaker.progress(generation)
    breaker.in_step = True
    try:
        yield
    finally:
        breaker.in_step = False
    if breaker.tripped:
        raise RuntimeError(f"the communicator was aborted while {what} was in flight")
