"""``aitjctl``: a kubectl-compatible CLI for the single-box control plane.

The reference's whole user workflow is four kubectl commands (/root/reference/README.md:14-19):
``kubectl apply -f job.yaml``, ``kubectl get aitj``, ``kubectl describe aitj <name>``,
``kubectl delete -f job.yaml``.  There is no kubectl in this environment (SURVEY.md Appendix C), so
this module re-implements that surface against the local API server with the same verbs, flags and
output shapes (SURVEY.md Appendix B): plain ``get`` prints ``NAME  AGE`` exactly like a CRD without
printer columns (controller.go:215-224), ``describe`` uses kubectl's generic describer layout
(humanised keys, nested 2-space indentation, Events table).  Extras that ``kubectl`` also has:
``-o yaml|json|wide|name``, ``-w``, ``-n`` / ``-A``, ``scale``, ``annotate``, ``patch``, ``edit``,
``logs``, ``api-resources``.  Fault injection for the BASELINE fail-over configs: ``aitjctl inject``.

    python -m trainingjob_operator_b200.cli.kubectl --server http://127.0.0.1:8001 get aitj
"""
from __future__ import annotations

import argparse
import json
import os
import re
import subprocess
import sys
import tempfile
import time
from typing import Any, Dict, List, Optional

import yaml

from ..api import constants as C
from ..api import meta as M
from ..api import register as R
from ..client.clientset import Clientset, new_for_config
from ..client.record import events_for
from ..cmd.options import TrainingJobOperatorOption, resolve_master
from ..store.apiserver import APIError

_ACRONYMS = {"api": "API", "url": "URL", "uid": "UID", "osb": "OSB", "guid": "GUID", "ip": "IP", "id": "ID"}


def humanize_key(key: str) -> str:
    """kubectl's ``smartLabelFor``: ``cleanPodPolicy`` -> ``Clean Pod Policy``, ``apiVersion`` -> ``API Version``."""
    if not key:
        return key
    if key.lower() in _ACRONYMS:
        return _ACRONYMS[key.lower()]
    parts = re.findall(r"[A-Z]+(?=[A-Z][a-z])|[A-Z]?[a-z0-9]+|[A-Z]+", key)
    if not parts:
        return key
    out = []
    for p in parts:
        lo = p.lower()
        out.append(_ACRONYMS.get(lo, p[:1].upper() + p[1:]))
    return " ".join(out)


def human_duration(seconds: float) -> str:
    """kubectl ``duration.HumanDuration``: 12s, 3m5s, 2h, 4d."""
    s = int(max(0, seconds))
    if s < 120:
        return f"{s}s"
    m = s // 60
    if m < 10:
        return f"{m}m{s % 60}s" if s % 60 else f"{m}m"
    if m < 180:
        return f"{m}m"
    h = m // 60
    if h < 8:
        return f"{h}h{m % 60}m" if m % 60 else f"{h}h"
    if h < 48:
        return f"{h}h"
    d = h // 24
    return f"{d}d"


def age_of(obj: Dict[str, Any]) -> str:
    ts = obj.get("metadata", {}).get("creationTimestamp")
    if not ts:
        return "<unknown>"
    return human_duration(M.seconds_since(ts))


def table(rows: List[List[str]]) -> str:
    if not rows:
        return ""
    widths = [max(len(str(r[i])) for r in rows) for i in range(len(rows[0]))]
    return "\n".join("   ".join(str(c).ljust(w) for c, w in zip(r, widths)).rstrip() for r in rows)


# ------------------------------------------------------------------------------------ describe
def _describe_value(lines: List[str], key: str, value: Any, indent: int) -> None:
    pad = "  " * indent
    label = humanize_key(key) + ":"
    if isinstance(value, dict):
        if not value:
            return
        lines.append(f"{pad}{label}")
        for k in sorted(value):
            _describe_value(lines, k, value[k], indent + 1)
    elif isinstance(value, list):
        if not value:
            return
        lines.append(f"{pad}{label}")
        for item in value:
            if isinstance(item, dict):
                first = True
                for k in sorted(item):
                    sub: List[str] = []
                    _describe_value(sub, k, item[k], indent + 1)
                    for s in sub:
                        lines.append(s)
                    first = False
                if first:
                    lines.append(f"{pad}  <empty>")
            else:
                lines.append(f"{pad}  {item}")
    else:
        if value is None:
            value = "<nil>"
        lines.append(f"{pad}{label}".ljust(len(pad) + len(label) + 2) + f"{value}")


def describe_object(obj: Dict[str, Any], events: Optional[List[Dict[str, Any]]] = None) -> str:
    md = obj.get("metadata", {})
    lines: List[str] = []

    def top(k: str, v: str) -> None:
        lines.append(f"{k + ':':<14}{v}")

    top("Name", md.get("name", ""))
    if md.get("namespace"):
        top("Namespace", md.get("namespace", ""))
    for title, mp in (("Labels", md.get("labels")), ("Annotations", md.get("annotations"))):
        if not mp:
            top(title, "<none>")
        else:
            items = [f"{k}={v}" if title == "Labels" else f"{k}: {v}" for k, v in sorted(mp.items())]
            top(title, items[0])
            for it in items[1:]:
                lines.append(" " * 14 + it)
    top("API Version", obj.get("apiVersion", ""))
    top("Kind", obj.get("kind", ""))
    rest_md = {k: v for k, v in md.items() if k not in ("name", "namespace", "labels", "annotations")}
    _describe_value(lines, "metadata", rest_md, 0)
    for k in sorted(obj):
        if k in ("apiVersion", "kind", "metadata"):
            continue
        _describe_value(lines, k, obj[k], 0)
    if events is not None:
        if not events:
            lines.append("Events:  <none>")
        else:
            lines.append("Events:")
            rows = [["  Type", "Reason", "Age", "From", "Message"], ["  ----", "------", "----", "----", "-------"]]
            for e in events:
                age = human_duration(M.seconds_since(e.get("lastTimestamp") or e.get("firstTimestamp")))
                if int(e.get("count", 1)) > 1:
                    age = f"{age} (x{e['count']} over {human_duration(M.seconds_since(e.get('firstTimestamp')))})"
                rows.append(["  " + e.get("type", ""), e.get("reason", ""), age,
                             (e.get("source") or {}).get("component", ""), e.get("message", "")])
            lines.append(table(rows))
    return "\n".join(lines)


# ------------------------------------------------------------------------------------ get
def get_rows(info: R.ResourceInfo, items: List[Dict[str, Any]], wide: bool, all_ns: bool) -> List[List[str]]:
    rows: List[List[str]] = []
    ns_col = ["NAMESPACE"] if all_ns else []
    if info.kind == C.KIND:
        hdr = ["NAME", "AGE"]
        if wide:
            hdr = ["NAME", "PHASE", "REPLICAS", "ACTIVE", "RESTARTS", "GENERATION", "AGE"]
        rows.append(ns_col + hdr)
        for o in items:
            st = o.get("status", {})
            if wide:
                specs = o.get("spec", {}).get("replicaSpecs", {})
                want = sum(int((s or {}).get("replicas", 1) or 0) for s in specs.values())
                active = sum(int((r or {}).get("active", 0)) for r in (st.get("replicaStatuses") or {}).values())
                restarts = max([0] + list((st.get("RestartCount") or {}).values()))
                gen = (st.get("rendezvous") or {}).get("generation", "")
                row = [M.name_of(o), st.get("phase", "") or "<none>", str(want), str(active), str(restarts), str(gen),
                       age_of(o)]
            else:
                row = [M.name_of(o), age_of(o)]
            rows.append(([M.namespace_of(o)] if all_ns else []) + row)
    elif info.kind == "Pod":
        rows.append(ns_col + ["NAME", "READY", "STATUS", "RESTARTS", "AGE"] + (["IP", "NODE", "GPUS"] if wide else []))
        for o in items:
            st = o.get("status", {})
            css = st.get("containerStatuses") or []
            n = len(o.get("spec", {}).get("containers") or [])
            ready = sum(1 for c in css if c.get("ready"))
            status = st.get("phase", "Pending")
            if o.get("metadata", {}).get("deletionTimestamp"):
                status = "Terminating"
            else:
                for c in css:
                    w = (c.get("state") or {}).get("waiting")
                    t = (c.get("state") or {}).get("terminated")
                    if w and w.get("reason"):
                        status = w["reason"]
                    elif t and t.get("exitCode", 0) != 0:
                        status = "Error"
                    elif t and status != "Error" and st.get("phase") == "Succeeded":
                        status = "Completed"
            row = [M.name_of(o), f"{ready}/{n}", status, M.labels_of(o).get(C.LABEL_RESTART_COUNT, "0"), age_of(o)]
            if wide:
                row += [st.get("podIP", "<none>"), o.get("spec", {}).get("nodeName", "<none>") or "<none>",
                        M.annotations_of(o).get(C.ANN_GPUS, "") or "<none>"]
            rows.append(([M.namespace_of(o)] if all_ns else []) + row)
    elif info.kind == "Service":
        rows.append(ns_col + ["NAME", "TYPE", "CLUSTER-IP", "PORT(S)", "AGE"])
        for o in items:
            ports = ",".join(f"{p.get('port')}/TCP" for p in o.get("spec", {}).get("ports") or []) or "<none>"
            rows.append(([M.namespace_of(o)] if all_ns else []) +
                        [M.name_of(o), "ClusterIP", o.get("spec", {}).get("clusterIP", ""), ports, age_of(o)])
    elif info.kind == "Node":
        rows.append(["NAME", "STATUS", "ROLES", "AGE", "VERSION"])
        for o in items:
            ready = any(c.get("type") == "Ready" and c.get("status") == "True"
                        for c in o.get("status", {}).get("conditions") or [])
            rows.append([M.name_of(o), "Ready" if ready else "NotReady", M.labels_of(o).get("aitj.b200/type", "<none>"),
                         age_of(o), o.get("status", {}).get("nodeInfo", {}).get("kubeletVersion", "")])
    elif info.kind == "Event":
        rows.append(ns_col + ["LAST SEEN", "TYPE", "REASON", "OBJECT", "MESSAGE"])
        for o in sorted(items, key=lambda e: e.get("lastTimestamp", "")):
            io = o.get("involvedObject", {})
            rows.append(([M.namespace_of(o)] if all_ns else []) +
                        [human_duration(M.seconds_since(o.get("lastTimestamp"))), o.get("type", ""), o.get("reason", ""),
                         f"{io.get('kind', '').lower()}/{io.get('name', '')}", o.get("message", "")])
    else:
        rows.append(ns_col + ["NAME", "AGE"])
        for o in items:
            rows.append(([M.namespace_of(o)] if all_ns and info.namespaced else []) + [M.name_of(o), age_of(o)])
    return rows


def dump(obj: Any, fmt: str) -> str:
    if fmt == "json":
        return json.dumps(obj, indent=4)
    return yaml.safe_dump(obj, sort_keys=False, default_flow_style=False).rstrip()


def load_manifests(path: str) -> List[Dict[str, Any]]:
    if path == "-":
        text = sys.stdin.read()
    elif path.startswith(("http://", "https://")):
        import urllib.request

        text = urllib.request.urlopen(path, timeout=10).read().decode()
    else:
        text = open(path).read()
    docs = [d for d in yaml.safe_load_all(text) if d]
    out = []
    for d in docs:
        if d.get("kind", "").endswith("List") and "items" in d:
            out += d["items"]
        else:
            out.append(d)
    return out


def parse_timeout(text: str) -> float:
    """``30s`` / ``2m`` / ``1h`` / bare seconds (kubectl's --timeout syntax); negative = a week."""
    t = text.strip()
    mult = {"s": 1.0, "m": 60.0, "h": 3600.0}.get(t[-1:], None)
    v = float(t[:-1]) if mult else float(t)
    v *= mult or 1.0
    return v if v >= 0 else 7 * 24 * 3600.0


def _wait_predicate(cond: str):
    """Predicate over the fetched object (None = not found) for ``wait --for=...``."""
    if cond == "delete":
        return lambda obj: obj is None
    kind, _, rest = cond.partition("=")
    if kind == "phase":
        return lambda obj: obj is not None and (obj.get("status") or {}).get("phase") == rest
    if kind == "condition":
        ctype, _, want = rest.partition("=")
        want = (want or "True").lower()

        def has_condition(obj) -> bool:
            if obj is None:
                return False
            last = None
            for c in (obj.get("status") or {}).get("conditions") or []:
                if str(c.get("type", "")).lower() == ctype.lower():
                    last = c                                      # the condition list is a history: the newest entry counts
            return last is not None and str(last.get("status", "")).lower() == want
        return has_condition
    if kind == "jsonpath":
        expr, _, want = rest.partition("=")
        path = [p for p in expr.strip("'\"{} ").split(".") if p]

        def at_path(obj) -> bool:
            cur: Any = obj
            for p in path:
                if not isinstance(cur, dict) or p not in cur:
                    return False
                cur = cur[p]
            return str(cur) == want.strip("'\"")
        return at_path
    raise RuntimeError(f"unrecognized condition: {cond!r} (use delete, phase=..., condition=..., jsonpath=...)")


# ------------------------------------------------------------------------------------ commands
class CLI:
    def __init__(self, cs: Clientset, out=sys.stdout):
        self.cs = cs
        self.out = out

    def p(self, s: str = "") -> None:
        print(s, file=self.out, flush=True)

    def _info(self, name: str) -> R.ResourceInfo:
        info = R.lookup(name)
        if info is None:
            raise APIError(404, "NotFound", f"the server doesn't have a resource type \"{name}\"")
        return info

    def _qualified(self, info: R.ResourceInfo) -> str:
        return f"{info.kind.lower()}.{info.group}" if info.group else info.kind.lower()

    def apply(self, files: List[str], namespace: str) -> int:
        for f in files:
            for obj in load_manifests(f):
                info = R.by_kind(obj["kind"])
                ns = obj.get("metadata", {}).get("namespace") or namespace
                rc = self.cs.resource(info, ns)
                name = M.name_of(obj)
                try:
                    cur = rc.get(name)
                except APIError as e:
                    if e.reason != "NotFound":
                        raise
                    if info.kind == C.KIND:
                        obj.setdefault("metadata", {}).setdefault("annotations", {}).setdefault(
                            C.ANN_TRACE, json.dumps({"submitted": round(time.time(), 4)}))
                    rc.create(obj)
                    self.p(f"{self._qualified(info)}/{name} created")
                    continue
                # like `kubectl apply`: merge the manifest onto the live object (server-side defaults survive)
                from ..store.apiserver import merge_patch

                desired = {k: v for k, v in obj.items() if k != "status"}
                md = dict(desired.get("metadata") or {})
                for k in ("resourceVersion", "uid", "creationTimestamp"):
                    md.pop(k, None)
                desired["metadata"] = md
                new = merge_patch(cur, desired)
                if new == cur:
                    self.p(f"{self._qualified(info)}/{name} unchanged")
                else:
                    rc.update(new)
                    self.p(f"{self._qualified(info)}/{name} configured")
        return 0

    def create(self, files: List[str], namespace: str) -> int:
        """``kubectl create -f``: like apply, but an existing object is an error (AlreadyExists)."""
        for f in files:
            for obj in load_manifests(f):
                info = R.by_kind(obj["kind"])
                ns = obj.get("metadata", {}).get("namespace") or namespace
                if info.kind == C.KIND:
                    obj.setdefault("metadata", {}).setdefault("annotations", {}).setdefault(
                        C.ANN_TRACE, json.dumps({"submitted": round(time.time(), 4)}))
                self.cs.resource(info, ns).create(obj)
                self.p(f"{self._qualified(info)}/{M.name_of(obj)} created")
        return 0

    def wait(self, resource: str, names: List[str], namespace: str, cond: str, timeout: float) -> int:
        """``kubectl wait --for=delete | --for=condition=<Type>[=True|False] | --for=jsonpath='{.a.b}'=value``, plus the
        shorthand ``--for=phase=<Phase>`` (``.status.phase``).  Exit 0 once every named object satisfies it, 1 on timeout."""
        if "/" in resource and not names:
            resource, n = resource.split("/", 1)
            names = [n]
        if not names:
            raise RuntimeError("wait needs a resource name (TYPE NAME or TYPE/NAME)")
        info = self._info(resource)
        rc = self.cs.resource(info, namespace)
        check = _wait_predicate(cond)
        deadline = time.monotonic() + timeout
        pending = list(names)
        while True:
            still = []
            for n in pending:
                try:
                    obj: Optional[Dict[str, Any]] = rc.get(n)
                except APIError as e:
                    if e.reason != "NotFound":
                        raise
                    obj = None
                if check(obj):
                    self.p(f"{self._qualified(info)}/{n} " + ("deleted" if obj is None else "condition met"))
                else:
                    still.append(n)
            pending = still
            if not pending:
                return 0
            if time.monotonic() > deadline:
                for n in pending:
                    print(f"error: timed out waiting for the condition on {info.plural}/{n}", file=sys.stderr)
                return 1
            time.sleep(0.05)

    def get(self, resource: str, names: List[str], namespace: str, all_ns: bool, output: str, watch: bool,
            selector: str) -> int:
        if "/" in resource and not names:
            resource, n = resource.split("/", 1)
            names = [n]
        info = self._info(resource)
        ns = "" if all_ns else namespace
        rc = self.cs.resource(info, ns)
        if names:
            items = [rc.get(n) for n in names]
            rv = ""
        else:
            lst = rc.list(selector)
            items, rv = lst["items"], lst["metadata"]["resourceVersion"]
        if output in ("yaml", "json"):
            if len(items) == 1 and names:
                self.p(dump(items[0], output))
            else:
                self.p(dump({"apiVersion": "v1", "kind": "List", "metadata": {"resourceVersion": ""}, "items": items},
                            output))
        elif output == "name":
            for o in items:
                self.p(f"{self._qualified(info)}/{M.name_of(o)}")
        else:
            if not items and not watch:
                scope = "" if all_ns or not info.namespaced else f" in {namespace} namespace"
                print(f"No resources found{scope}.", file=sys.stderr)
            else:
                self.p(table(get_rows(info, items, output == "wide", all_ns)))
        if watch:
            try:
                for ev in rc.watch(resource_version=rv, label_selector=selector):
                    o = ev["object"]
                    if names and M.name_of(o) not in names:
                        continue
                    if output in ("yaml", "json"):
                        self.p(dump(o, output))
                    else:
                        rows = get_rows(info, [o], output == "wide", all_ns)
                        self.p(table(rows[1:]))
            except KeyboardInterrupt:
                pass
        return 0

    def describe(self, resource: str, names: List[str], namespace: str) -> int:
        if "/" in resource and not names:
            resource, n = resource.split("/", 1)
            names = [n]
        info = self._info(resource)
        rc = self.cs.resource(info, namespace)
        objs = [rc.get(n) for n in names] if names else rc.list()["items"]
        for i, o in enumerate(objs):
            if i:
                self.p("\n")
            try:
                evs = events_for(self.cs, o)
            except APIError:
                evs = []
            self.p(describe_object(o, evs))
        return 0

    def delete(self, resource: Optional[str], names: List[str], files: List[str], namespace: str, grace: Optional[int],
               all_: bool) -> int:
        targets = []
        for f in files:
            for obj in load_manifests(f):
                targets.append((R.by_kind(obj["kind"]), obj.get("metadata", {}).get("namespace") or namespace,
                                M.name_of(obj)))
        if resource:
            if "/" in resource and not names:
                resource, n = resource.split("/", 1)
                names = [n]
            info = self._info(resource)
            if all_:
                names = [M.name_of(o) for o in self.cs.resource(info, namespace).list()["items"]]
            targets += [(info, namespace, n) for n in names]
        rc_code = 0
        for info, ns, name in targets:
            try:
                self.cs.resource(info, ns).delete(name, grace)
                self.p(f"{self._qualified(info)} \"{name}\" deleted")
            except APIError as e:
                print(f"Error from server ({e.reason}): {e.message}", file=sys.stderr)
                rc_code = 1
        return rc_code

    def scale(self, resource: str, name: str, namespace: str, replicas: int, role: Optional[str]) -> int:
        info = self._info(resource)
        if "/" in name:
            name = name.split("/", 1)[1]
        obj = self.cs.resource(info, namespace).get(name)
        specs = obj.get("spec", {}).get("replicaSpecs", {})
        if role is None:
            if len(specs) != 1:
                raise APIError(400, "BadRequest", f"job has roles {sorted(specs)}; pass --role")
            role = next(iter(specs))
        self.cs.resource(info, namespace).patch(name, {"spec": {"replicaSpecs": {role: {"replicas": replicas}}}})
        self.p(f"{self._qualified(info)}/{name} scaled")
        return 0

    def annotate(self, resource: str, name: str, namespace: str, pairs: List[str], overwrite: bool) -> int:
        info = self._info(resource)
        ann: Dict[str, Optional[str]] = {}
        for kv in pairs:
            if kv.endswith("-"):
                ann[kv[:-1]] = None
            else:
                k, v = kv.split("=", 1)
                ann[k] = v
        cur = self.cs.resource(info, namespace).get(name)
        if not overwrite:
            for k, v in ann.items():
                if v is not None and k in M.annotations_of(cur) and M.annotations_of(cur)[k] != v:
                    raise APIError(400, "BadRequest", f"--overwrite is false but found the following declared "
                                   f"annotation(s): '{k}' already has a value ({M.annotations_of(cur)[k]})")
        self.cs.resource(info, namespace).patch(name, {"metadata": {"annotations": ann}})
        self.p(f"{self._qualified(info)}/{name} annotated")
        return 0

    def patch(self, resource: str, name: str, namespace: str, patch: str, ptype: str) -> int:
        info = self._info(resource)
        body = yaml.safe_load(patch)
        ctype = {"merge": "application/merge-patch+json", "json": "application/json-patch+json",
                 "strategic": "application/merge-patch+json"}[ptype]
        self.cs.resource(info, namespace).patch(name, body, ctype)
        self.p(f"{self._qualified(info)}/{name} patched")
        return 0

    def edit(self, resource: str, name: str, namespace: str) -> int:
        info = self._info(resource)
        rc = self.cs.resource(info, namespace)
        cur = rc.get(name)
        with tempfile.NamedTemporaryFile("w+", suffix=".yaml", delete=False) as f:
            f.write(dump(cur, "yaml") + "\n")
            path = f.name
        editor = os.environ.get("KUBE_EDITOR") or os.environ.get("EDITOR") or "vi"
        subprocess.call(editor.split() + [path])
        new = yaml.safe_load(open(path))
        os.unlink(path)
        if new == cur:
            self.p("Edit cancelled, no changes made.")
            return 0
        rc.update(new)
        self.p(f"{self._qualified(info)}/{name} edited")
        return 0

    def logs(self, pod: str, namespace: str, container: Optional[str], workdir: str, tail: Optional[int],
             follow: bool) -> int:
        obj = self.cs.core_v1().pods(namespace).get(pod)
        names = [c["name"] for c in obj.get("spec", {}).get("containers") or []]
        cname = container or (names[0] if names else "")
        path = os.path.join(workdir, "logs", f"{namespace}_{pod}_{cname}.log")
        if not os.path.exists(path):
            print(f"log file {path} not found (is --workdir the agent's workdir?)", file=sys.stderr)
            return 1
        with open(path) as f:
            lines = f.readlines()
            for ln in (lines[-tail:] if tail else lines):
                self.out.write(ln)
            while follow:
                ln = f.readline()
                if ln:
                    self.out.write(ln)
                    self.out.flush()
                else:
                    time.sleep(0.2)
        return 0

    def api_resources(self) -> int:
        rows = [["NAME", "SHORTNAMES", "APIVERSION", "NAMESPACED", "KIND"]]
        for r in sorted(R.all_resources(), key=lambda r: r.plural):
            rows.append([r.plural, ",".join(r.short_names), r.api_version, str(r.namespaced).lower(), r.kind])
        self.p(table(rows))
        return 0

    def top(self, namespace: str, all_ns: bool) -> int:
        """``kubectl top``'s place in this world: what the jobs' rank-0 workers last reported (``aitj.b200/metrics``,
        ``aitj.b200/rescale-trace``) -- throughput, step time, world size, in-place recoveries, HellaSwag accuracy,
        held-out loss."""
        jobs = self.cs.elasticdeeplearning_v1().aitrainingjobs("" if all_ns else namespace).list().items
        rows = [["NAME", "PHASE", "WORLD", "SAMPLES/S", "MS/STEP", "STEPS", "RECOVERIES", "LAST RESCALE", "HELLASWAG",
                 "EVAL LOSS"]]
        for j in jobs:
            try:
                m = json.loads(j.annotations.get("aitj.b200/metrics", "{}")) or {}
                r = json.loads(j.annotations.get("aitj.b200/rescale-trace", "{}")) or {}
            except ValueError:
                m, r = {}, {}
            world = sum((j.status.rendezvous.world_sizes or {}).values()) if j.status.rendezvous else ""
            rows.append([j.name, j.status.phase or "<none>", str(world or "<none>"),
                         f"{m['samples_per_sec']:.1f}" if m.get("samples_per_sec") else "<none>",
                         f"{m['ms_per_step']:.2f}" if m.get("ms_per_step") else "<none>",
                         str(m.get("steps_done", "<none>")), str(m.get("recoveries", 0)),
                         f"{r['seconds']:.2f}s -> world {r.get('world')}" if r.get("seconds") else "<none>",
                         f"{m['hellaswag_acc']:.4f}" if m.get("hellaswag_acc") is not None else "<none>",
                         f"{m['eval_loss']:.4f}" if m.get("eval_loss") is not None else "<none>"])
        if len(rows) == 1:
            self.p("No resources found.")
            return 0
        self.p(table(rows))
        return 0

    def inject(self, what: str, target: str, namespace: str, value: str) -> int:
        """Fault injection: ``gpu-fault gpu-3`` / ``gpu-heal gpu-3`` mark a GPU slot NotReady / Ready;
        ``preempt <job>`` / ``fail <job>`` write the external control annotations (pod.go:160-165)."""
        if what in ("gpu-fault", "gpu-heal"):
            ann = {C.ANN_INJECT_FAULT: (value or "injected fault") if what == "gpu-fault" else None}
            self.cs.core_v1().nodes().patch(target, {"metadata": {"annotations": ann}})
            self.p(f"node/{target} {'marked faulty' if what == 'gpu-fault' else 'healed'}")
        elif what in ("preempt", "fail"):
            key = C.PHASE_PREEMPTED if what == "preempt" else C.PHASE_FAILED
            self.cs.resource(R.AITRAININGJOB, namespace).patch(
                target, {"metadata": {"annotations": {key: value or f"{what} requested by aitjctl"}}})
            self.p(f"aitrainingjob.{C.GROUP_NAME}/{target} annotated {key}")
        else:
            raise APIError(400, "BadRequest", f"unknown injection {what}")
        return 0


def build_parser() -> argparse.ArgumentParser:
    ap = argparse.ArgumentParser(prog="aitjctl", description="kubectl-compatible CLI for AITrainingJobs")
    ap.add_argument("--server", "-s", default="", help="API server URL (default: ~/.aitj/config or $AITJ_MASTER)")
    ap.add_argument("--kubeconfig", default="")
    ap.add_argument("--namespace", "-n", default="default")
    sub = ap.add_subparsers(dest="cmd", required=True)

    def common(p):
        p.add_argument("--namespace", "-n", dest="ns2", default=None)

    a = sub.add_parser("apply"); a.add_argument("-f", "--filename", action="append", required=True); common(a)
    cr = sub.add_parser("create"); cr.add_argument("-f", "--filename", action="append", required=True); common(cr)
    wt = sub.add_parser("wait"); wt.add_argument("resource"); wt.add_argument("names", nargs="*")
    wt.add_argument("--for", dest="cond", required=True); wt.add_argument("--timeout", default="30s"); common(wt)
    g = sub.add_parser("get"); g.add_argument("resource"); g.add_argument("names", nargs="*")
    g.add_argument("-o", "--output", default=""); g.add_argument("-w", "--watch", action="store_true")
    g.add_argument("-A", "--all-namespaces", action="store_true"); g.add_argument("-l", "--selector", default="")
    common(g)
    d = sub.add_parser("describe"); d.add_argument("resource"); d.add_argument("names", nargs="*"); common(d)
    x = sub.add_parser("delete"); x.add_argument("resource", nargs="?"); x.add_argument("names", nargs="*")
    x.add_argument("-f", "--filename", action="append", default=[]); x.add_argument("--grace-period", type=int)
    x.add_argument("--force", action="store_true"); x.add_argument("--all", action="store_true"); common(x)
    s = sub.add_parser("scale"); s.add_argument("resource"); s.add_argument("name", nargs="?")
    s.add_argument("--replicas", type=int, required=True); s.add_argument("--role"); common(s)
    n = sub.add_parser("annotate"); n.add_argument("resource"); n.add_argument("name"); n.add_argument("pairs", nargs="+")
    n.add_argument("--overwrite", action="store_true"); common(n)
    pt = sub.add_parser("patch"); pt.add_argument("resource"); pt.add_argument("name")
    pt.add_argument("-p", "--patch", required=True); pt.add_argument("--type", default="merge",
                                                                      choices=["merge", "json", "strategic"]); common(pt)
    e = sub.add_parser("edit"); e.add_argument("resource"); e.add_argument("name"); common(e)
    lg = sub.add_parser("logs"); lg.add_argument("pod"); lg.add_argument("-c", "--container")
    lg.add_argument("--workdir", default=os.path.expanduser("~/.aitj")); lg.add_argument("--tail", type=int)
    lg.add_argument("-f", "--follow", action="store_true"); common(lg)
    tp = sub.add_parser("top"); tp.add_argument("resource", nargs="?", default="aitj")
    tp.add_argument("-A", "--all-namespaces", action="store_true"); common(tp)
    sub.add_parser("api-resources")
    sub.add_parser("version")
    sub.add_parser("cluster-info")
    ij = sub.add_parser("inject"); ij.add_argument("what", choices=["gpu-fault", "gpu-heal", "preempt", "fail"])
    ij.add_argument("target"); ij.add_argument("--message", default=""); common(ij)
    return ap


def main(argv=None, clientset: Optional[Clientset] = None, out=sys.stdout) -> int:
    parser = build_parser()
    args, extra = parser.parse_known_args(argv)
    if extra:
        # kubectl accepts flags anywhere (`wait aitj --for=delete NAME`); argparse stops collecting a `nargs="*"` positional at
        # the first flag, so names that follow flags arrive here
        if any(e.startswith("-") for e in extra) or not hasattr(args, "names"):
            parser.error("unrecognized arguments: " + " ".join(extra))
        args.names = list(args.names) + extra
    ns = getattr(args, "ns2", None) or args.namespace
    try:
        if clientset is None:
            master = resolve_master(TrainingJobOperatorOption(master_url=args.server, kubeconfig=args.kubeconfig))
            clientset = new_for_config(master=master)
        cli = CLI(clientset, out)
        if args.cmd == "apply":
            return cli.apply(args.filename, ns)
        if args.cmd == "create":
            return cli.create(args.filename, ns)
        if args.cmd == "wait":
            return cli.wait(args.resource, args.names, ns, args.cond, parse_timeout(args.timeout))
        if args.cmd == "get":
            return cli.get(args.resource, args.names, ns, args.all_namespaces, args.output, args.watch, args.selector)
        if args.cmd == "describe":
            return cli.describe(args.resource, args.names, ns)
        if args.cmd == "delete":
            grace = 0 if args.force else args.grace_period
            return cli.delete(args.resource, args.names, args.filename, ns, grace, args.all)
        if args.cmd == "scale":
            res, name = args.resource, args.name
            if name is None and "/" in res:
                res, name = res.split("/", 1)
            return cli.scale(res, name, ns, args.replicas, args.role)
        if args.cmd == "annotate":
            return cli.annotate(args.resource, args.name, ns, args.pairs, args.overwrite)
        if args.cmd == "patch":
            return cli.patch(args.resource, args.name, ns, args.patch, args.type)
        if args.cmd == "edit":
            return cli.edit(args.resource, args.name, ns)
        if args.cmd == "logs":
            return cli.logs(args.pod, ns, args.container, args.workdir, args.tail, args.follow)
        if args.cmd == "top":
            return cli.top(ns, args.all_namespaces)
        if args.cmd == "api-resources":
            return cli.api_resources()
        if args.cmd == "version":
            cli.p("Client Version: aitjctl v0.1.0\nServer Version: v1.13.5-aitj-b200")
            return 0
        if args.cmd == "cluster-info":
            cli.p(f"AITrainingJob control plane is running at {getattr(clientset.transport, 'master', 'in-process')}")
            return 0
        if args.cmd == "inject":
            return cli.inject(args.what, args.target, ns, args.message)
    except APIError as e:
        print(f"Error from server ({e.reason}): {e.message}", file=sys.stderr)
        return 1
    except (RuntimeError, FileNotFoundError, ValueError) as e:
        print(f"error: {e}", file=sys.stderr)
        return 1
    return 0


if __name__ == "__main__":
    sys.exit(main())
