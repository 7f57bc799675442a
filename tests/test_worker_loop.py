"""The result record of ``runtime/worker.py run()``, end to end on one CPU rank: its exact keys and the timed region's
step accounting, which ``bench.py`` and the controller's reports read."""
import json
import os
import subprocess
import sys
import textwrap

import pytest

from test_packed_documents import structured_corpus, write_llmc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTS = os.path.dirname(os.path.abspath(__file__))

BASE_KEYS = {"rank", "world", "steps_done", "generation", "final_loss", "rescales", "recoveries", "trace"}
TIMED_KEYS = {"timed_steps", "timed_from_step", "timed_region_epoch", "ms_per_step", "samples_per_sec",
              "wall_ms_per_step", "global_batch", "batch_per_gpu", "micro_batches", "micro_batches_this_rank",
              "h2d_bytes_per_step", "d2h_bytes_per_step", "gpu_launches", "launches_per_step", "loss_first",
              "loss_last", "flops_per_step", "describe", "cuda_graph", "graph_segments", "graph_error", "allreduce"}

# the GPT-2 engine adapter on the CPU: kernel entry points emulated (tests/kernel_emulation.py)
ENGINE_WORKER = """
import sys
sys.path.insert(0, {root!r}); sys.path.insert(0, {tests!r})
import kernel_emulation as ke
ke.install()
from trainingjob_operator_b200.runtime import worker as W
W.build_adapter = lambda args, device: W.EngineAdapter(args.model, args.batch, args.seq, args, device="cpu")
sys.exit(W.main(sys.argv[1:]))
"""


def _run(tmp_path, argv, script=None):
    """One rank, no control plane; returns the result record rank 0 wrote."""
    result = tmp_path / "result.json"
    if script is None:
        cmd = [sys.executable, "-m", "trainingjob_operator_b200.runtime.worker"]
    else:
        path = tmp_path / "worker.py"
        path.write_text(textwrap.dedent(script.format(root=ROOT, tests=TESTS)))
        cmd = [sys.executable, str(path)]
    env = dict(os.environ, RANK="0", WORLD_SIZE="1", OMP_NUM_THREADS="2", AITJ_WORKDIR=str(tmp_path),
               PYTHONPATH=ROOT)
    for k in ("AITJ_MASTER", "TRAININGJOB_REPLICA_RESTARTCOUNT", "AITJ_FAULT_TOLERANT"):
        env.pop(k, None)
    p = subprocess.run(cmd + ["--cpu", "--result", str(result)] + argv, env=env, cwd=ROOT, capture_output=True,
                       text=True, timeout=600)
    assert p.returncode == 0, (p.stdout + p.stderr)[-4000:]
    return json.load(open(result))


def _check_timed(r, steps, warmup):
    assert r["timed_steps"] == steps and r["timed_from_step"] == warmup and r["steps_done"] == warmup + steps, r
    t0, t1 = r["timed_region_epoch"]
    assert 0 < t0 <= t1, r["timed_region_epoch"]
    assert r["world"] == 1 and r["generation"] == 0 and r["rescales"] == [] and r["recoveries"] == []
    assert r["ms_per_step"] > 0 and r["wall_ms_per_step"] > 0 and r["samples_per_sec"] > 0


def test_result_record_of_a_timed_nn_module_run(tmp_path):
    r = _run(tmp_path, ["--model", "mlp", "--batch", "8", "--steps", "4", "--warmup", "2"])
    assert set(r) == BASE_KEYS | TIMED_KEYS, sorted(set(r) ^ (BASE_KEYS | TIMED_KEYS))
    assert len(r) == 30
    _check_timed(r, 4, 2)
    assert r["global_batch"] == 8 and r["batch_per_gpu"] == 8 and r["micro_batches"] == 1
    assert r["micro_batches_this_rank"] == 1 and r["h2d_bytes_per_step"] == 8 * 64 * 4 + 8 * 8
    assert r["cuda_graph"] is False and r["graph_segments"] is None and r["graph_error"] is None
    assert r["allreduce"] == "none" and r["launches_per_step"] == 0 and r["gpu_launches"] == 0


@pytest.mark.slow
def test_result_record_of_a_gpt2_run_with_held_out_evaluation(tmp_path):
    train = write_llmc(tmp_path / "train_000.bin", structured_corpus(20000, 1000, 999, 3))
    val = write_llmc(tmp_path / "val_000.bin", structured_corpus(8000, 1000, 999, 4))
    r = _run(tmp_path, ["--model", "gpt2-tiny", "--batch", "2", "--seq", "128", "--steps", "4", "--warmup", "2",
                        "--data", train, "--eval-data", val, "--eval-every", "2", "--eval-samples", "3"], ENGINE_WORKER)
    assert set(r) == BASE_KEYS | TIMED_KEYS | {"data_position", "evals", "eval_loss_last"}, sorted(r)
    _check_timed(r, 4, 2)
    assert r["data_position"] == 6 * 2
    assert [e["step"] for e in r["evals"]] == [2, 4, 6]
    assert all(set(e) == {"step", "loss", "tokens", "samples", "ms"} for e in r["evals"])
    assert r["eval_loss_last"] == r["evals"][-1]["loss"]
