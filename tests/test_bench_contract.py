"""bench.py's CPU arm (`--impl reference`) runs without a GPU: check that it prints ONE JSON line with the contract's keys.
(The GPU arm is exercised by the driver; its extra keys are listed here so that a rename shows up in review.)"""
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BASE_KEYS = {"metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline",
             "dtype", "data", "config"}
GPU_ARM_KEYS = BASE_KEYS | {"clocks", "e2e", "gpu_launches", "roofline", "cpu_baseline"}


def test_reference_arm_prints_the_contract_line():
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--cpu-rows", "4000", "--trees", "4",
                          "--depth", "4", "--steps", "1", "--warmup", "1"], capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-2000:]
    lines = [l for l in out.stdout.splitlines() if l.startswith("{")]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert BASE_KEYS <= set(d) and d["impl"] == "reference" and d["higher_is_better"] is True and d["vs_baseline"] is None
    assert d["unit"] == "records/s" and d["value"] > 0 and "workload" in d["config"]
    assert {"value", "unit", "cores", "kind", "sample"} <= set(d["cpu_baseline"]) and d["cpu_baseline"]["kind"] == "port"
    assert d["e2e"]["h2d_bytes_per_step"] == 0 and d["e2e"]["d2h_bytes_per_step"] == 0 and d["e2e"]["value"] == d["value"]


def test_reference_arm_sets_its_thread_count_and_honours_warmup():
    # torchrun exports OMP_NUM_THREADS=1 to its workers: the CPU arm must not inherit it (the N>1 arms would time out)
    env = dict(os.environ, OMP_NUM_THREADS="1", RANK="0", WORLD_SIZE="2")
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--gpus", "2", "--workload", "cicids_script",
                          "--cpu-rows", "3000", "--trees", "3", "--depth", "3", "--steps", "1", "--warmup", "2"],
                         capture_output=True, text=True, timeout=600, cwd=ROOT, env=env)
    assert out.returncode == 0, out.stderr[-2000:]
    d = json.loads([l for l in out.stdout.splitlines() if l.startswith("{")][0])
    cores = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else os.cpu_count()
    assert d["cpu_baseline"]["cores"] == cores and d["warmup"] == 2 and d["n_gpus"] == 2
    assert d["config"]["name"] == "cicids_script" and d["config"]["sample_rows"] == 3000 and d["config"]["classes"] == 14


def test_reference_arm_other_ranks_exit_quietly():
    env = dict(os.environ, RANK="1", WORLD_SIZE="2")
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--gpus", "2", "--steps", "1"],
                         capture_output=True, text=True, timeout=300, cwd=ROOT, env=env)
    assert out.returncode == 0 and out.stdout.strip() == ""


def test_gpu_arm_keys_are_emitted_by_bench_source():
    src = open(os.path.join(ROOT, "bench.py")).read()
    for k in GPU_ARM_KEYS | {"traffic", "frac", "peak", "achieved", "bound", "h2d_bytes_per_step", "d2h_bytes_per_step", "sm_mhz",
                             "dram_frac", "lsu_pct", "labels_equal", "forest_equal", "forest_hash"}:
        assert '"%s"' % k in src, k


def _dump(path):
    subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--cpu-rows", "3000", "--trees", "3",
                    "--depth", "4", "--steps", "2", "--warmup", "0", "--dump-outputs", str(path)], capture_output=True, text=True, check=True)
    return {f: np.load(os.path.join(path, f)) for f in sorted(os.listdir(path))}


def test_reference_arm_dumps_identical_float64_outputs(tmp_path):
    a, b = _dump(tmp_path / "a"), _dump(tmp_path / "b")
    assert {"prediction.npy", "macro_f1.npy", "forest_nodes.npy", "forest_counts.npy", "forest_masks.npy"} <= set(a)
    assert a.keys() == b.keys() and all(a[k].dtype == np.float64 and np.array_equal(a[k], b[k]) for k in a)
    assert sum(os.path.getsize(tmp_path / "a" / f) for f in a) <= 60 << 20


def test_reference_dump_needs_a_fixed_batch(tmp_path):
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--dump-outputs", str(tmp_path)],
                         capture_output=True, text=True)
    assert out.returncode != 0 and "--cpu-rows" in out.stderr


def test_dump_outputs_samples_rows_beyond_the_budget(tmp_path):
    sys.path.insert(0, ROOT)
    import bench
    arrays = {"big": np.arange(40000, dtype=np.float64).reshape(-1, 4), "small": np.arange(3, dtype=np.int32), "f": 0.5}
    for d in ("a", "b"):
        bench.dump_outputs(str(tmp_path / d), arrays, budget=1 << 16)
    files = sorted(os.listdir(tmp_path / "a"))
    assert files == ["big.npy", "big_rows.npy", "f.npy", "small.npy"] and sum(os.path.getsize(tmp_path / "a" / f) for f in files) <= 1 << 16
    rows, big = np.load(tmp_path / "a" / "big_rows.npy"), np.load(tmp_path / "a" / "big.npy")
    assert big.dtype == np.float64 and np.all(np.diff(rows) > 0) and np.array_equal(big, arrays["big"][rows.astype(np.int64)])
    assert np.array_equal(np.load(tmp_path / "a" / "small.npy"), [0.0, 1.0, 2.0]) and np.load(tmp_path / "a" / "f.npy").tolist() == [0.5]
    assert all(np.array_equal(np.load(tmp_path / "a" / f), np.load(tmp_path / "b" / f)) for f in files)
