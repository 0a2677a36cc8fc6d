"""bench.py prints ONE JSON line with the keys the driver reads (CPU: reference arm; GPU: b200 arm)."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BASE_KEYS = {"metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
             "vs_baseline", "dtype", "data", "config"}


def _run(args, timeout=600):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py")] + args, capture_output=True, text=True,
                       timeout=timeout, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [l for l in r.stdout.splitlines() if l.startswith("{")]
    assert len(lines) == 1, r.stdout
    return json.loads(lines[0])


def test_reference_arm_line():
    d = _run(["--impl", "reference", "--workload", "mnist_cnn", "--steps", "8", "--warmup", "3", "--cpu-budget", "1"])
    assert BASE_KEYS <= set(d) and d["impl"] == "reference" and d["higher_is_better"] is True
    assert d["unit"] == "micro-steps/s" and d["value"] > 0 and d["vs_baseline"] is None and d["dtype"] == "f32"
    assert "workload" in d["config"] and "model" not in d["config"]
    cb = d["cpu_baseline"]
    assert cb["kind"] == "port" and cb["cores"] >= 1 and cb["value"] == d["value"] and cb["sample"]
    assert d["e2e"] == {"value": d["value"], "unit": d["unit"], "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}


def test_reference_arm_nonzero_rank_prints_nothing():
    env = dict(os.environ, RANK="1", WORLD_SIZE="2", LOCAL_RANK="1")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--gpus", "2"],
                       capture_output=True, text=True, timeout=120, cwd=ROOT, env=env)
    assert r.returncode == 0 and r.stdout.strip() == ""


@pytest.mark.gpu
def test_b200_arm_line():
    d = _run(["--workload", "mnist_cnn", "--steps", "40", "--warmup", "3", "--e2e-steps", "8", "--cpu-budget", "1"])
    assert BASE_KEYS <= set(d) and d["impl"] == "b200" and d["n_gpus"] == 1 and d["steps"] == 40 and d["warmup"] >= 3
    assert d["scaling"] == "weak" and d["data"] == "synthetic" and d["dtype"] == "f32" and d["gpu_launches"] == 40
    rf = d["roofline"]
    assert {"bound", "achieved", "peak", "unit", "frac", "traffic"} <= set(rf) and rf["bound"] == "hbm" and rf["unit"] == "GB/s"
    assert abs(rf["frac"] - rf["achieved"] / rf["peak"]) < 1e-9
    e = d["e2e"]
    assert e["value"] > 0 and e["h2d_bytes_per_step"] == 4 * d["config"]["P"] and e["d2h_bytes_per_step"] > 0
    assert {"sm_mhz", "sm_max_mhz", "reasons"} <= set(d["clocks"])
    assert d["cpu_baseline"]["kind"] == "port" and d["cpu_baseline"]["value"] > 0
    assert "l2" in d["config"] and "workload" in d["config"]
    # exact window mix: 40 steps at N=4 are 10 applies + 30 accumulates, and the line says so
    assert d["config"]["apply_launches"] == 10 and d["config"]["accumulate_launches"] == 30 and d["config"]["window_exact"] is True
    # the pre-timing parity self-check ran against the oracle and passed
    assert d["parity"]["ok"] is True and d["parity"]["max_rel_err"] <= 1e-5 and d["parity"]["world"] == 1


def test_both_arms_print_the_same_metric_string():
    """The driver divides the two arms only when `metric` matches: one constant feeds both lines."""
    import re
    src = open(os.path.join(ROOT, "bench.py")).read()
    assert len(re.findall(r'"metric": METRIC', src)) >= 2 and '"impl": "b200"' in src and '"impl": "reference"' in src


@pytest.mark.parametrize("N", [1, 2, 3, 4, 5, 6, 8, 32])
def test_rotation_phases_give_one_apply_per_window(N):
    """bench.py steps R rotating state sets round-robin; the per-set global_step phases must put exactly one
    apply (pre-increment step % N == 0, optimization.py:91) at bench steps i % N == N-1 and nowhere else."""
    sys.path.insert(0, ROOT)
    import bench
    R = bench.rotation_for(N)
    assert R >= 3
    gs = [bench.set_start_step(r, R, N) for r in range(R)]
    for i in range(6 * N * R):
        r = i % R
        applies = (gs[r] % N) == 0
        gs[r] += 1
        assert applies == (i % N == N - 1), (N, R, i)


def test_dump_outputs_writes_the_packed_state_sampled_at_fixed_positions(tmp_path, monkeypatch):
    """dump_outputs on a stand-in op (CPU tensors): one float .npy per array, tensors packed without the slab padding,
    every array sampled at the same seeded positions, and the whole dump within 64 MB at the real sample size."""
    import numpy as np
    import torch
    sys.path.insert(0, ROOT)
    import bench

    class Plan:
        offsets = [0, 32, 64]                       # slab offsets: tensors padded to 32 elements
    sizes = [5, 20, 7]
    slab = lambda k: torch.arange(96, dtype=torch.float32) + 1000 * k
    op = type("Op", (), {"plan": Plan(), "accum": slab(1), "m": slab(2), "v": slab(3),
                         "stats": lambda self: {"applied": True, "lr": 0.5, "global_norm": 2.0, "clip_scale": 0.25}})()
    params = [torch.full((n,), float(i)) for i, n in enumerate(sizes)]
    packed = lambda s: np.concatenate([s.numpy()[o:o + n] for o, n in zip(Plan.offsets, sizes)])
    want = {"params": np.concatenate([p.numpy() for p in params]), "accum": packed(slab(1)),
            "adam_m": packed(slab(2)), "adam_v": packed(slab(3))}

    monkeypatch.setattr(bench, "DUMP_SAMPLE", 10)
    bench.dump_outputs(str(tmp_path / "a"), op, params, None)
    bench.dump_outputs(str(tmp_path / "b"), op, params, None)
    files = sorted(os.listdir(tmp_path / "a"))
    assert files == ["accum.npy", "adam_m.npy", "adam_v.npy", "params.npy", "sample_index.npy", "stats.npy"]
    idx = np.load(tmp_path / "a" / "sample_index.npy")
    assert idx.dtype == np.float64 and len(idx) == 10 and np.all(np.diff(idx) > 0) and idx.max() < sum(sizes)
    for f in files:
        a, b = np.load(tmp_path / "a" / f), np.load(tmp_path / "b" / f)
        assert a.dtype in (np.float32, np.float64) and np.array_equal(a, b), f      # same inputs -> same dump
    for name, full in want.items():
        assert np.array_equal(np.load(tmp_path / "a" / f"{name}.npy"), full[idx.astype(np.int64)]), name
    assert np.array_equal(np.load(tmp_path / "a" / "stats.npy"), np.array([1.0, 0.5, 2.0, 0.25], np.float32))

    monkeypatch.setattr(bench, "DUMP_SAMPLE", 1000)                   # fewer elements than the sample: all of them
    bench.dump_outputs(str(tmp_path / "c"), op, params, None)
    assert np.array_equal(np.load(tmp_path / "c" / "sample_index.npy"), np.arange(sum(sizes), dtype=np.float64))
    monkeypatch.undo()
    assert 4 * 4 * bench.DUMP_SAMPLE + 8 * bench.DUMP_SAMPLE + 16 <= 64 << 20


@pytest.mark.gpu
def test_b200_arm_dumps_what_the_last_timed_step_computed(tmp_path):
    """--dump-outputs writes the state set the last timed micro-step used: after an apply step its accumulators are
    all zero (the other sets are mid-window), after an accumulate step they are not; the same arguments give the same dump."""
    import numpy as np
    lean = ["--workload", "mnist_cnn", "--warmup", "3", "--model-steps", "0", "--e2e-steps", "0", "--cpu-budget", "0",
            "--parity-steps", "0"]
    for K, tag in ((40, "a"), (40, "b"), (42, "c")):
        _run(lean + ["--steps", str(K), "--dump-outputs", str(tmp_path / tag)])
    load = lambda tag, name: np.load(tmp_path / tag / f"{name}.npy")
    for name in ("params", "accum", "adam_m", "adam_v", "sample_index", "stats"):
        assert np.array_equal(load("a", name), load("b", name)), name
    assert load("a", "stats")[0] == 1.0 and not load("a", "accum").any()         # step 39 of N=4 applies
    assert load("c", "stats")[0] == 0.0 and load("c", "accum").any()             # step 41 accumulates
