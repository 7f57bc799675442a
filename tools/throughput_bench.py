"""Control-plane throughput (no GPU needed): J jobs x R replicas of a trivial command submitted at once through the
public API; time until every job is Succeed, jobs/s and pods/s, API-server write count, reconcile latency.  Run once
with the default reconcile-queue bucket and once with client-go's 10 qps / burst 100 (what the reference inherits).

    python tools/throughput_bench.py [jobs] [replicas] [thread_num]   -> profiles/control_plane_throughput.json
"""
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from trainingjob_operator_b200.api import constants as C  # noqa: E402
from trainingjob_operator_b200.cmd.local import LocalCluster  # noqa: E402
from trainingjob_operator_b200.cmd.options import TrainingJobOperatorOption  # noqa: E402
from trainingjob_operator_b200.utils import klog, metrics  # noqa: E402


def job(name, replicas):
    c = {"name": "aitj-trainer", "command": ["/bin/true"]}
    return {"apiVersion": C.API_VERSION, "kind": C.KIND, "metadata": {"name": name},
            "spec": {"cleanPodPolicy": "All",
                     "replicaSpecs": {"trainer": {"replicas": replicas, "template": {"spec": {"containers": [c]}}}}}}


def run(jobs, replicas, threads, **opt_kw):
    opt = TrainingJobOperatorOption(thread_num=threads, **opt_kw)
    with LocalCluster(num_gpus=0, option=opt) as lc:
        klog.set_verbosity(-1)
        import logging
        logging.getLogger("aitj").setLevel(logging.ERROR)
        rv0 = int(lc.clientset.core_v1().pods("default").list()["metadata"]["resourceVersion"] or 0)
        t0 = time.perf_counter()
        for i in range(jobs):
            lc.apply(job(f"tp-{i}", replicas))
        t_submitted = time.perf_counter() - t0
        done_at = {}
        deadline = time.time() + 600
        # completion is read from the raw objects every 50 ms: a typed list of every job every 10 ms made the observer the
        # second largest consumer of the interpreter lock in the process it measures
        raw = lc.jobs().raw
        while len(done_at) < jobs and time.time() < deadline:
            for j in raw.list().get("items", []):
                name = j["metadata"]["name"]
                if name not in done_at and (j.get("status") or {}).get("phase") == "Succeed":
                    done_at[name] = time.perf_counter() - t0
            time.sleep(0.05)
        total = time.perf_counter() - t0
        rv1 = int(lc.clientset.core_v1().pods("default").list()["metadata"]["resourceVersion"] or 0)
        lat = sorted(done_at.values())
        out = {"jobs": jobs, "replicas": replicas, "thread_num": threads, "completed": len(done_at),
               "submit_all_s": round(t_submitted, 3), "all_succeed_s": round(total, 3),
               "jobs_per_s": round(len(done_at) / total, 1), "pods_per_s": round(len(done_at) * replicas / total, 1),
               "store_writes": rv1 - rv0, "writes_per_s": round((rv1 - rv0) / total, 1),
               "job_latency_p50_s": round(lat[len(lat) // 2], 3) if lat else None,
               "job_latency_p99_s": round(lat[min(len(lat) - 1, int(0.99 * len(lat)))], 3) if lat else None}
        return out


def run_daemons(jobs, replicas, threads):
    """The README topology: API server, node agent and operator as three processes talking HTTP on loopback."""
    import socket
    import subprocess
    import tempfile

    from trainingjob_operator_b200.client.clientset import new_for_config

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    wd = tempfile.mkdtemp(prefix="aitj-tp-")
    env = dict(os.environ, PYTHONPATH=root)
    procs = []

    def spawn(mod, *args):
        procs.append(subprocess.Popen([sys.executable, "-m", f"trainingjob_operator_b200.cmd.{mod}", *args], cwd=root,
                                      env=env, stdout=open(os.path.join(wd, f"{mod}.log"), "w"),
                                      stderr=subprocess.STDOUT))

    try:
        spawn("apiserver", "--port", str(port), "--data-dir", os.path.join(wd, "data"))
        cs = new_for_config(master=f"127.0.0.1:{port}")
        jobs_api = cs.elasticdeeplearning_v1().aitrainingjobs("default")
        for _ in range(200):
            try:
                jobs_api.list()
                break
            except Exception:  # noqa: BLE001
                time.sleep(0.1)
        spawn("agent", "--master", f"127.0.0.1:{port}", "--gpus", "0", "--workdir", os.path.join(wd, "agent"),
              "--warm-pool", "0")
        spawn("main", "--master", f"127.0.0.1:{port}", "--thread-num", str(threads))
        time.sleep(2.0)
        from trainingjob_operator_b200.api.types import AITrainingJob

        t0 = time.perf_counter()
        for i in range(jobs):
            jobs_api.create(AITrainingJob.from_dict(job(f"tp-{i}", replicas)))
        t_submitted = time.perf_counter() - t0
        done_at = {}
        deadline = time.time() + 900
        while len(done_at) < jobs and time.time() < deadline:
            for j in jobs_api.list().items:
                if j.name not in done_at and j.status.phase == "Succeed":
                    done_at[j.name] = time.perf_counter() - t0
            time.sleep(0.05)
        total = time.perf_counter() - t0
        lat = sorted(done_at.values())
        cpu = {}
        try:
            import psutil

            for name, p in zip(("apiserver", "agent", "operator"), procs):
                t = psutil.Process(p.pid).cpu_times()
                cpu[name] = round(t.user + t.system, 2)
        except Exception:  # noqa: BLE001
            pass
        # single-job latency in the same topology: submit -> phase Running, 8 replicas of /bin/sleep
        single = []
        for i in range(10):
            jd = job(f"one-{i}", replicas)
            jd["spec"]["replicaSpecs"]["trainer"]["template"]["spec"]["containers"][0]["command"] = ["/bin/sleep", "600"]
            t1 = time.perf_counter()
            jobs_api.create(AITrainingJob.from_dict(jd))
            while jobs_api.get(f"one-{i}").status.phase != "Running":
                time.sleep(0.001)
            single.append(time.perf_counter() - t1)
            jobs_api.delete(f"one-{i}")
            time.sleep(0.3)
        single.sort()
        return {"topology": "3 processes over loopback HTTP",
                "submit_to_running_p50_s": round(single[len(single) // 2], 4),
                "submit_to_running_max_s": round(single[-1], 4), "cpu_seconds_until_all_succeed": cpu, "jobs": jobs, "replicas": replicas, "thread_num": threads,
                "completed": len(done_at), "submit_all_s": round(t_submitted, 3), "all_succeed_s": round(total, 3),
                "jobs_per_s": round(len(done_at) / total, 1), "pods_per_s": round(len(done_at) * replicas / total, 1),
                "job_latency_p50_s": round(lat[len(lat) // 2], 3) if lat else None,
                "job_latency_p99_s": round(lat[min(len(lat) - 1, int(0.99 * len(lat)))], 3) if lat else None}
    finally:
        for p in reversed(procs):
            p.terminate()
        for p in procs:
            try:
                p.wait(10)
            except subprocess.TimeoutExpired:
                p.kill()


def main():
    if "--daemons" in sys.argv:
        sys.argv.remove("--daemons")
        jobs = int(sys.argv[1]) if len(sys.argv) > 1 else 50
        replicas = int(sys.argv[2]) if len(sys.argv) > 2 else 8
        threads = int(sys.argv[3]) if len(sys.argv) > 3 else 8
        out = run_daemons(jobs, replicas, threads)
        print(json.dumps(out), flush=True)
        path = "profiles/control_plane_throughput.json"
        d = json.load(open(path)) if os.path.exists(path) else {}
        d["three_daemons_http"] = out
        os.makedirs("profiles", exist_ok=True)
        json.dump(d, open(path, "w"), indent=1)
        return
    jobs = int(sys.argv[1]) if len(sys.argv) > 1 else 100
    replicas = int(sys.argv[2]) if len(sys.argv) > 2 else 8
    threads = int(sys.argv[3]) if len(sys.argv) > 3 else 8
    path = "profiles/control_plane_throughput.json"
    out = json.load(open(path)) if os.path.exists(path) else {}      # keeps the history sections and the daemon run
    out["default_queue"] = run(jobs, replicas, threads)
    print(json.dumps(out["default_queue"]), flush=True)
    out["client_go_queue_10qps_burst100"] = run(jobs, replicas, threads, queue_qps=10.0, queue_burst=100)
    print(json.dumps(out["client_go_queue_10qps_burst100"]), flush=True)
    out["note"] = ("each job: create R pods + R services, bind + start + reap R processes, status writes, delete pods + "
                   "services (cleanPodPolicy All), final condition.  The reference additionally sits behind client-go's "
                   "5 qps / burst 10 REST throttle per clientset (SURVEY.md 2.2), which is not modelled here.")
    os.makedirs("profiles", exist_ok=True)
    json.dump(out, open(path, "w"), indent=1)


if __name__ == "__main__":
    main()
