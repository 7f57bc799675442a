"""Job event handlers and worker-report metrics.

What the reference does on job events (/root/reference/pkg/controller/trainingjob.go:17-51): add -> enqueue now,
update with a new resourceVersion -> enqueue rate-limited plus a delayed enqueue when ``timeLimit`` changed, delete ->
enqueue.  Its two ``// FIXME: need to validate trainingjob`` (:21,:33) are resolved: invalid objects are rejected at
admission and, defensively, skipped here with a warning.  Naming (:12-15) lives in ``pod.gen_general_name``; the
teardown of a finished job (:53-73, and quirk Q9: services leaked when there were no pods) is part of the engine's
``terminate`` decision.
"""
from __future__ import annotations

from ..api import meta as M
from ..api.validation import validate_dict
from ..utils import klog, metrics

# what the workers report back onto the job (runtime/elastic.py) becomes scrapeable (SURVEY.md §5.5: rescale latency and
# per-job samples/sec belong on /metrics; the reference has no metrics at all)
ANN_WORKER_METRICS = "aitj.b200/metrics"
ANN_WORKER_RESCALE = "aitj.b200/rescale-trace"
metrics.describe("aitj_rescale_seconds", "membership change observed by the workers -> first step at the new world "
                                         "(kind=rescale|recovery)")
metrics.describe("aitj_job_samples_per_second", "whole-job training throughput reported by rank 0")
metrics.describe("aitj_job_eval_loss", "mean held-out loss per token of the job's last evaluation, reported by rank 0")
metrics.describe("aitj_job_hellaswag_acc", "HellaSwag accuracy of the job's last scoring, reported by rank 0")
metrics.describe("aitj_job_recoveries_total", "in-place recoveries of faultTolerant jobs (a rank was lost, the others kept "
                                              "their state)")


def observe_worker_reports(old: dict, cur: dict) -> None:
    """Turn changed worker-report annotations into metrics (called from the job update handler)."""
    import json

    a_old, a_cur = M.annotations_of(old), M.annotations_of(cur)
    labels = {"namespace": M.namespace_of(cur) or "default", "job": M.name_of(cur)}
    raw = a_cur.get(ANN_WORKER_RESCALE)
    if raw and raw != a_old.get(ANN_WORKER_RESCALE):
        try:
            rec = json.loads(raw)
            kind = "recovery" if rec.get("recovered_from") else "rescale"
            metrics.observe("aitj_rescale_seconds", float(rec["seconds"]), labels={"kind": kind})
            if kind == "recovery":
                metrics.inc("aitj_job_recoveries_total", labels=labels)
        except (ValueError, KeyError, TypeError):
            pass
    raw = a_cur.get(ANN_WORKER_METRICS)
    if raw and raw != a_old.get(ANN_WORKER_METRICS):
        try:
            rec = json.loads(raw)
            v = rec.get("samples_per_sec")
            if v is not None:
                metrics.set_gauge("aitj_job_samples_per_second", float(v), labels=labels)
            v = rec.get("eval_loss")
            if v is not None:
                metrics.set_gauge("aitj_job_eval_loss", float(v), labels=labels)
            v = rec.get("hellaswag_acc")
            if v is not None:
                metrics.set_gauge("aitj_job_hellaswag_acc", float(v), labels=labels)
        except (ValueError, TypeError, AttributeError):
            pass


class TrainingJobHandlers:
    """Mixed into ``TrainingJobController``."""

    def add_training_job(self, obj: dict) -> None:
        klog.V(2).info("Informer: Add TrainingJob %s/%s.", M.namespace_of(obj), M.name_of(obj))
        errs = validate_dict(obj)
        if errs:
            klog.warning("TrainingJob %s/%s is invalid, not reconciling: %s", M.namespace_of(obj), M.name_of(obj),
                         "; ".join(errs))
            return
        self.enqueue_job(obj, False, 0)

    def update_training_job(self, old: dict, cur: dict) -> None:
        if M.resource_version(old) == M.resource_version(cur):
            klog.V(4).info("Same Resourceversion for training job %s/%s, skipped", M.namespace_of(old),
                           M.name_of(old))
            return
        errs = validate_dict(cur)
        if errs:
            klog.warning("TrainingJob %s/%s is invalid, not reconciling: %s", M.namespace_of(cur), M.name_of(cur),
                         "; ".join(errs))
            return
        klog.V(2).info("Informer: Update TrainingJob %s/%s.", M.namespace_of(old), M.name_of(old))
        observe_worker_reports(old, cur)
        spec_changed = old.get("spec") != cur.get("spec") or \
            M.annotations_of(old) != M.annotations_of(cur)
        # a spec/annotation edit by the user is acted on immediately; our own status writes are rate limited
        self.enqueue_job(cur, not spec_changed, 0)
        new_limit = cur.get("spec", {}).get("timeLimit")
        old_limit = old.get("spec", {}).get("timeLimit")
        started = cur.get("status", {}).get("startRunningTime")
        if started and new_limit is not None and new_limit != old_limit:
            remaining = int(new_limit) - int(M.seconds_since(started))
            self.enqueue_job(cur, False, max(remaining, 0) + 0.05)
            klog.info("job TimeLimit updated, will rsync after %d seconds", remaining)

    def delete_training_job(self, obj) -> None:
        self.enqueue_job(obj, False, 0)
