"""The kernel launches of one GPT-2 and one BERT training step, pinned against ``tests/golden/engine_launches.json``.

Under the kernel emulation every entry point of ``ops.functional`` is wrapped, and one ``forward()``, ``backward()`` and
``optimizer_step()`` is recorded in order: the entry point, every tensor argument as its buffer, offset, dtype and
shape, and every other argument as its value.  Buffers are numbered by first use among the storages the engine owns
(parameters, gradients, optimizer state and the activations it allocates); any other tensor, such as an SDPA
temporary, is ``tmp``.  The trace therefore follows the aliasing between launches and not allocator addresses: a change
to the engines' host code that keeps this file unchanged issues the same work to the GPU.

    python tests/test_engine_launches.py        # re-record, for a change that alters the launches on purpose
"""
import inspect
import json
import os
import sys
import threading

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import kernel_emulation as ke  # noqa: E402
from trainingjob_operator_b200.ops import functional as F  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "engine_launches.json")
ENV = ("AITJ_ATTN", "AITJ_ATTN_BWD", "AITJ_GEMM_PAIR", "AITJ_GEMM_CFG", "AITJ_WGRAD_STREAM")
# the library's entry points, taken before any test replaces them: their signatures name every argument of a call
ENTRY_POINTS = {n: inspect.signature(f) for n, f in vars(F).items()
                if inspect.isfunction(f) and f.__module__ == F.__name__ and not n.startswith("_")}

# name -> (model, constructor keywords, environment, owner-sharded)
CONFIGS = {
    "gpt2": ("gpt2", {}, {}, False),
    "gpt2-attn-wgmma": ("gpt2", {}, {"AITJ_ATTN": "wgmma", "AITJ_ATTN_BWD": "wgmma"}, False),
    "gpt2-no-pair": ("gpt2", {}, {"AITJ_GEMM_PAIR": "0"}, False),
    "gpt2-cublas": ("gpt2", {"gemm_backend": "cublas"}, {}, False),
    "gpt2-doc-mask": ("gpt2", {"doc_mask": True}, {}, False),
    "gpt2-owner-sharded": ("gpt2", {}, {}, True),
    "bert": ("bert", {}, {}, False),
    "bert-owner-sharded": ("bert", {}, {}, True),
}


def _engine(model, kw):
    if model == "gpt2":
        from trainingjob_operator_b200.models.gpt2 import GPT2Config, GPT2Engine

        cfg = GPT2Config(vocab_size=1000, n_layer=2, n_head=4, n_embd=256, block_size=128, name="t")
        return GPT2Engine(cfg, 2, 128, "cpu", seed=3, **kw)
    from trainingjob_operator_b200.models.bert import BertConfig, BertEngine

    return BertEngine(BertConfig.tiny(), 2, 128, "cpu", seed=3, **kw)


def _owned_storages(eng):
    """Every tensor reachable from the engine's attributes (layers, parameters, shard buffers), by storage pointer."""
    out, seen = {}, set()

    def walk(x):
        if id(x) in seen:
            return
        seen.add(id(x))
        if isinstance(x, torch.Tensor):
            out[x.untyped_storage().data_ptr()] = x
        elif isinstance(x, (list, tuple)):
            for y in x:
                walk(y)
        elif type(x).__module__.split(".")[0] in ("trainingjob_operator_b200", "kernel_emulation"):
            for y in vars(x).values():
                walk(y)

    walk(eng)
    return out


class _Recorder:
    def __init__(self, eng):
        # holding the tensors keeps their addresses from being reused by temporaries, such as the SDPA output that
        # ``att_in`` still points to from the previous step
        self.owned = _owned_storages(eng)
        self.ids = {}
        self.calls = []
        self.thread = threading.get_ident()
        shard = eng.params.shard
        # a pointer token whose value depends on how many emulated worlds the process created before
        self.aliases = {shard.parts_mc: "parts_mc"} if shard is not None else {}

    def tensor(self, t):
        s = t.untyped_storage().data_ptr()
        if s in self.owned:
            buf = f"b{self.ids.setdefault(s, len(self.ids))}@{t.storage_offset()}"
        else:
            buf = "tmp"
        d = f"{buf}:{str(t.dtype).replace('torch.', '')}{list(t.shape)}"
        return d if t.is_contiguous() else d + f"/{list(t.stride())}"

    def value(self, v):
        if isinstance(v, torch.Tensor):
            return self.tensor(v)
        if isinstance(v, F.PeerView):
            return "peer:" + self.tensor(v.t)
        if isinstance(v, int) and not isinstance(v, bool) and v in self.aliases:
            return self.aliases[v]
        assert v is None or isinstance(v, (bool, int, float, str)), type(v)
        return v

    def wrap(self, name, fn):
        sig = ENTRY_POINTS[name]

        def entry(*a, **k):
            if threading.get_ident() == self.thread:
                bound = sig.bind(*a, **k)
                bound.apply_defaults()
                self.calls.append([name, {p: self.value(v) for p, v in bound.arguments.items()}])
            return fn(*a, **k)

        return entry


def _step(eng):
    eng.forward()
    eng.backward()
    eng.optimizer_step(lr=1e-3, step=1)


def trace(name, mp):
    """The launches of one step of configuration ``name`` (after an untimed step that allocates the lazy buffers)."""
    from test_packed_documents import install_doc_attention

    model, kw, env, sharded = CONFIGS[name]
    install_doc_attention(mp)
    for k in ENV:
        mp.delenv(k, raising=False)
    for k, v in env.items():
        mp.setenv(k, v)
    eng = _engine(model, kw)
    peers = []
    if sharded:
        fw = ke.FakeWorld(2)
        mp.setitem(ke._CURRENT, "world", fw)
        peers = [_engine(model, kw)]
        fw.attach(eng.params)
        fw.attach(peers[0].params)
    errors = []

    def run(e, rec=None):
        try:
            _step(e)
            if rec is not None:
                rec.append(_Recorder(e))
                for n in ENTRY_POINTS:
                    mp.setattr(F, n, rec[0].wrap(n, getattr(F, n)))
            _step(e)
        except Exception as ex:  # noqa: BLE001
            errors.append(repr(ex))
            if sharded:
                fw.sync.abort()

    rec = []
    if not sharded:
        run(eng, rec)
    else:
        # the ranks meet at barriers inside the optimizer step, so each runs in its own thread; rank 0 is recorded
        threads = [threading.Thread(target=run, args=(e, r)) for e, r in ((eng, rec), (peers[0], None))]
        for t in threads:
            t.start()
        for t in threads:
            t.join(600)
    assert not errors, errors
    return rec[0].calls


def _dump(traces):
    parts = []
    for name, calls in traces.items():
        rows = ",\n".join("    " + json.dumps(c) for c in calls)
        parts.append(f"  {json.dumps(name)}: [\n{rows}\n  ]")
    return "{\n" + ",\n".join(parts) + "\n}\n"


@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_engine_step_issues_the_recorded_launches(monkeypatch, name):
    with open(GOLDEN) as f:
        want = json.load(f)[name]
    got = trace(name, monkeypatch)
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, f"launch {i} of {len(want)} differs:\n got  {g}\n want {w}"
    assert len(got) == len(want), (len(got), len(want))


if __name__ == "__main__":
    traces = {}
    for n in CONFIGS:
        with pytest.MonkeyPatch.context() as mp:
            traces[n] = trace(n, mp)
    with open(GOLDEN, "w") as f:
        f.write(_dump(traces))
    print(f"{GOLDEN}: {', '.join(f'{n} {len(c)}' for n, c in traces.items())} launches")
