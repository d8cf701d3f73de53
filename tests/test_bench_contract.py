"""bench.py's driver-facing contract that can be checked without a GPU: the reference arm prints one JSON
line with the agreed keys, and the product arm refuses to run without CUDA (no CPU fallback)."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def run(*args, env=None):
    e = dict(os.environ)
    e.pop("RANK", None); e.pop("WORLD_SIZE", None); e.pop("LOCAL_RANK", None)
    if env:
        e.update(env)
    return subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), *args], capture_output=True, text=True,
                          timeout=600, cwd=ROOT, env=e)


def test_reference_arm_json_line():
    r = run("--impl", "reference", "--queries", "2", "--steps", "1", "--warmup", "1")
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [l for l in r.stdout.splitlines() if l.strip()]
    assert len(lines) == 1, r.stdout  # exactly one line on stdout
    d = json.loads(lines[0])
    assert d["impl"] == "reference"
    for k in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
              "vs_baseline", "dtype", "data", "config", "cpu_baseline", "e2e"):
        assert k in d, k
    assert d["unit"] == "UIDs/s" and d["higher_is_better"] is True and d["vs_baseline"] is None
    assert d["steps"] == 1 and d["warmup"] == 1 and d["value"] > 0 and d["ms_per_step"] > 0
    assert "workload" in d["config"] and "model" not in d["config"]
    cb = d["cpu_baseline"]
    assert cb["kind"] in ("port", "reference") and cb["cores"] >= 1 and cb["sample"] and cb["value"] == d["value"]
    assert cb["cores"] == min(2, os.cpu_count())  # the threads that are actually busy: one per query
    e2e = d["e2e"]
    assert e2e["value"] == d["value"] and e2e["unit"] == d["unit"]
    assert e2e["h2d_bytes_per_step"] == 0 and e2e["d2h_bytes_per_step"] == 0


def test_reference_arm_same_config_at_n_gpus():
    """At N GPUs the reference arm runs the whole job's N x Q queries on rank 0 and reports the GPU arm's config."""
    r = run("--impl", "reference", "--gpus", "2", "--queries", "2", "--steps", "1", "--warmup", "1",
            env={"RANK": "0", "LOCAL_RANK": "0", "WORLD_SIZE": "2"})
    assert r.returncode == 0, r.stderr[-2000:]
    d = json.loads(r.stdout.strip())
    assert d["n_gpus"] == 2 and d["config"]["queries_per_gpu"] == 2
    assert "2 GPU(s)" in d["config"]["parallelism"]
    assert d["cpu_baseline"]["cores"] == min(4, os.cpu_count())
    assert "4 queries (2 x 2)" in d["cpu_baseline"]["sample"]


def test_reference_arm_other_ranks_exit_quietly():
    r = run("--impl", "reference", "--gpus", "2", "--queries", "2", "--steps", "1", "--warmup", "0",
            env={"RANK": "1", "LOCAL_RANK": "1", "WORLD_SIZE": "2"})
    assert r.returncode == 0 and r.stdout.strip() == ""


def test_reference_arm_refuses_dump_outputs(tmp_path):
    r = run("--impl", "reference", "--queries", "2", "--steps", "1", "--dump-outputs", str(tmp_path / "d"))
    assert r.returncode != 0 and "--dump-outputs" in r.stderr
    assert not (tmp_path / "d").exists()


def _bench_module():
    import importlib.util

    spec = importlib.util.spec_from_file_location("bench_under_test", os.path.join(ROOT, "bench.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _result_buffer(q, values):
    """bench.py's result buffer layout: [out_off (q+1 words) | values | 2 words of slack], int64."""
    import numpy as np
    import torch

    rng = np.random.default_rng(7)
    cuts = np.sort(rng.integers(0, values.size + 1, q - 1))
    off = np.concatenate([[0], cuts, [values.size]]).astype(np.uint64)
    host = np.concatenate([off, values, np.array([123, 456], np.uint64)])
    return torch.from_numpy(host.view(np.int64)), off


def test_dump_outputs_writes_offsets_and_uids(tmp_path):
    import numpy as np

    bench = _bench_module()
    vals = np.cumsum(np.arange(1, 1001, dtype=np.uint64))
    buf, off = _result_buffer(5, vals)
    bench.dump_outputs(str(tmp_path), buf, 5, 0, 1)
    assert sorted(p.name for p in tmp_path.iterdir()) == ["offsets.npy", "uids.npy"]
    o, u = np.load(tmp_path / "offsets.npy"), np.load(tmp_path / "uids.npy")
    assert o.dtype == np.float64 and u.dtype == np.float64
    assert np.array_equal(o, off.astype(np.float64)) and np.array_equal(u, vals.astype(np.float64))


def test_dump_outputs_samples_past_the_budget(tmp_path, monkeypatch):
    import numpy as np

    bench = _bench_module()
    monkeypatch.setattr(bench, "DUMP_BYTES", 8 * 1024)
    vals = np.cumsum(np.arange(1, 5001, dtype=np.uint64))
    buf, off = _result_buffer(3, vals)
    for d in ("a", "b"):
        bench.dump_outputs(str(tmp_path / d), buf, 3, 0, 1)
    a = {n: np.load(tmp_path / "a" / f"{n}.npy") for n in ("offsets", "uids", "uids_index")}
    b = {n: np.load(tmp_path / "b" / f"{n}.npy") for n in ("offsets", "uids", "uids_index")}
    assert all(np.array_equal(a[n], b[n]) for n in a)          # the sample is fixed
    assert sum(x.nbytes for x in a.values()) <= 8 * 1024
    idx = a["uids_index"].astype(np.int64)
    assert idx.size > 0 and np.all(np.diff(idx) > 0)
    assert np.array_equal(a["uids"], vals[idx].astype(np.float64))
    assert np.array_equal(a["offsets"], off.astype(np.float64))


def test_product_arm_needs_cuda():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    r = run("--steps", "1", "--warmup", "0", "--queries", "1")
    assert r.returncode != 0
    assert "CUDA" in (r.stderr + r.stdout)
