"""CPU: the reference arm of bench.py (the one arm that runs without a GPU) prints exactly one JSON line with the keys a
consumer of the bench reads; the GPU arm's shape is checked on the committed H100 line (profiles/bench_h100.json)."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(*extra):
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--N", "9", "--Nsub", "20",
                          "--cpu-seeds", "2", "--steps", "1", "--warmup", "1", *extra], capture_output=True, text=True,
                         timeout=600, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-2000:]
    lines = [l for l in out.stdout.splitlines() if l.startswith("{")]
    assert len(lines) == 1
    return json.loads(lines[0])


def test_reference_arm_json_line():
    d = _run()
    for k in ("impl", "metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
              "vs_baseline", "dtype", "data", "config", "cpu_baseline", "e2e"):
        assert k in d, k
    assert d["impl"] == "reference" and d["higher_is_better"] is True and d["dtype"] == "f64" and d["data"] == "synthetic"
    assert d["value"] > 0 and d["cpu_baseline"]["kind"] == "port" and d["cpu_baseline"]["cores"] >= 1
    assert d["e2e"]["h2d_bytes_per_step"] == 0 and d["e2e"]["d2h_bytes_per_step"] == 0
    assert "starship_flip PTR" in d["config"]["workload"]


def test_reference_arm_other_ranks_are_silent():
    env = dict(os.environ, RANK="1", WORLD_SIZE="2", LOCAL_RANK="1")
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--gpus", "2", "--N", "9",
                          "--Nsub", "20", "--cpu-seeds", "2", "--steps", "1", "--warmup", "1"], capture_output=True,
                         text=True, timeout=300, cwd=ROOT, env=env)
    assert out.returncode == 0 and not [l for l in out.stdout.splitlines() if l.startswith("{")]


DUMP_SCRIPT = """
import sys, types
import numpy as np
sys.path.insert(0, sys.argv[1])
import bench
B, N = 40, 5
rng = np.random.default_rng(1)
sol = types.SimpleNamespace(xd=rng.standard_normal((B, N, 3)), ud=rng.standard_normal((B, N, 2)),
                            p=rng.standard_normal((B, 4)), cost=rng.standard_normal(B), deviation=rng.standard_normal(B),
                            iterations=np.arange(B, dtype=np.int32), feas=np.ones(B, dtype=np.int32),
                            raw_status=np.zeros(B, dtype=np.int32), td=np.linspace(0.0, 1.0, N))
bench.dump_outputs(sol, sys.argv[2] + "/full")
SEED_BYTES = 8 * (5 * 3 + 5 * 2 + 4 + 5 + 1)     # one seed's results and its entry in seed_index.npy
bench.DUMP_BYTES = 12 * SEED_BYTES + 8 * N         # room for 12 seeds and the time grid
bench.dump_outputs(sol, sys.argv[2] + "/sample")
"""


def _dump(out_dir):
    r = subprocess.run([sys.executable, "-c", DUMP_SCRIPT, ROOT, str(out_dir)], capture_output=True, text=True,
                       timeout=120, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]


def test_dump_outputs_writes_every_result_array_and_samples_above_the_limit(tmp_path):
    """--dump-outputs: the per-seed results of the timed path as float64 .npy files; over the size limit a fixed seeded
    sample of the seeds, the same on every run, with the sampled seed numbers beside it."""
    import numpy as np
    _dump(tmp_path / "a")
    _dump(tmp_path / "b")
    names = {"xd", "ud", "p", "cost", "deviation", "iterations", "feas", "status", "td"}
    assert {f.stem for f in (tmp_path / "a" / "full").iterdir()} == names
    full = {n: np.load(tmp_path / "a" / "full" / f"{n}.npy") for n in names}
    assert all(a.dtype == np.float64 for a in full.values())
    assert full["xd"].shape == (40, 5, 3) and np.array_equal(full["iterations"], np.arange(40))
    sample = {f.stem: np.load(f) for f in (tmp_path / "a" / "sample").iterdir()}
    assert set(sample) == names | {"seed_index"}
    idx = sample["seed_index"].astype(int)
    assert len(idx) == 12 and np.all(np.diff(idx) > 0)
    assert np.array_equal(idx, np.load(tmp_path / "b" / "sample" / "seed_index.npy"))
    assert sum(a.nbytes for a in sample.values()) <= 12 * 8 * 35 + 8 * 5
    for n in names - {"td"}:
        assert np.array_equal(sample[n], full[n][idx])


def test_committed_gpu_bench_line_has_the_contract_keys():
    d = json.load(open(os.path.join(ROOT, "profiles", "bench_h100.json")))
    for k in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
              "vs_baseline", "dtype", "data", "config", "gpu_launches", "e2e", "roofline", "cpu_baseline", "clocks"):
        assert k in d, k
    r = d["roofline"]
    assert r["bound"] == "hbm" and abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-12 and r["unit"] == "GB/s"
    assert d["gpu_launches"] > 0 and d["e2e"]["h2d_bytes_per_step"] > 0 and d["warmup"] >= 3
    k1 = d["roofline_k1"]
    assert k1["bound"] == "fp64" and k1["unit"] == "TFLOP/s" and abs(k1["frac"] - k1["achieved"] / k1["peak"]) < 1e-12
    assert d["cpu_baseline"]["kind"] == "port" and d["cpu_baseline"]["cores"] >= 1 and d["clocks"]["reasons"] == []
    assert set(d["config"]) == {"workload", "batch_total", "batch_per_gpu", "partition", "algorithm_constants", "seeds", "l2"}
