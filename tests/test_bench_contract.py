"""The JSON line bench.py prints, checked key by key: on live GPU runs of every configuration and on a live run of the CPU
reference arm."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BASE = {"metric": str, "value": (int, float), "unit": str, "n_gpus": int, "steps": int, "warmup": int, "ms_per_step": (int, float),
        "higher_is_better": bool, "scaling": str, "dtype": str, "data": str, "config": dict}


def _check_common(j):
    for k, t in BASE.items():
        assert k in j and isinstance(j[k], t), (k, j.get(k))
    assert "vs_baseline" in j and j["vs_baseline"] is None           # BASELINE.md holds no published number for this metric
    assert "workload" in j["config"] and not ({"model", "seq_len", "global_batch"} & set(j["config"]))
    e = j["e2e"]
    assert set(e) >= {"value", "unit", "h2d_bytes_per_step", "d2h_bytes_per_step"} and e["unit"] == j["unit"]


GPU_RUNS = {"lv": ["--n-per-gpu", "16384", "--no-strong"], "seir": ["--n-per-gpu", "4096"], "fkpp": ["--n-per-gpu", "1024"], "hjb": ["--n-per-gpu", "2000"]}


@pytest.mark.gpu
@pytest.mark.parametrize("config", sorted(GPU_RUNS))
def test_gpu_bench_line(config, tmp_path):
    """One GPU run of bench.py per configuration: the JSON line, and the arrays --dump-outputs writes after the timed steps."""
    dump = tmp_path / "out"
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--config", config, "--steps", "4", "--warmup", "2",
                          "--cpu-sample", "64", "--dump-outputs", str(dump)] + GPU_RUNS[config], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stderr[-2000:]
    j = json.loads([l for l in out.stdout.splitlines() if l.startswith("{")][-1])
    _check_common(j)
    assert j["steps"] == 4 and j["n_gpus"] == 1
    assert j["value"] > 0 and j["gpu_launches"] > 0 and j["e2e"]["value"] > 0
    assert j["e2e"]["h2d_bytes_per_step"] > 0 and j["e2e"]["d2h_bytes_per_step"] > 0 and abs(j["e2e"]["value"] - j["value"]) > 0
    r = j["roofline"]
    assert r["bound"] in ("hbm", "tensor") and r["unit"] in ("GB/s", "TFLOP/s") and set(r) >= {"achieved", "peak", "frac", "traffic"}
    assert abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-9 and 0 < r["frac"] <= 1
    c = j["clocks"]
    assert set(c) >= {"sm_mhz", "sm_max_mhz", "reasons"} and not ({"hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown"} & set(c["reasons"]))
    assert j["gpu"]["name"] and j["gpu"]["power_limit_w"] > 0
    b = j["cpu_baseline"]
    assert set(b) >= {"value", "unit", "cores", "kind", "sample"} and b["kind"] in ("port", "reference") and b["cores"] >= 1
    files = {f.stem: np.load(f) for f in dump.iterdir()}
    want = {"theta", "loss_history", "u0_history"} if config == "hjb" else {"out", "grad_theta", "loss"}
    assert want <= set(files) and sum(f.stat().st_size for f in dump.iterdir()) <= 64 * 10**6
    assert all(a.dtype in (np.float32, np.float64) and np.isfinite(a).all() for a in files.values())


@pytest.mark.parametrize("extra", [["--n-per-gpu", "1024"], ["--config", "hjb", "--n-per-gpu", "200"]])
def test_reference_arm_live(extra):
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "3", "--warmup", "1"] + extra,
                         capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    j = json.loads([l for l in out.stdout.splitlines() if l.startswith("{")][-1])
    _check_common(j)
    assert j["impl"] == "reference" and j["value"] > 0
    assert j["e2e"]["value"] == j["value"] and j["e2e"]["h2d_bytes_per_step"] == 0 and j["e2e"]["d2h_bytes_per_step"] == 0
    b = j["cpu_baseline"]
    assert b["kind"] == "port" and b["value"] == j["value"] and b["cores"] >= 1 and isinstance(b["sample"], str)


def test_reference_arm_other_ranks_exit_quietly():
    env = dict(os.environ, RANK="1", WORLD_SIZE="2", LOCAL_RANK="1")
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--gpus", "2", "--n-per-gpu", "512"],
                         capture_output=True, text=True, timeout=300, env=env)
    assert out.returncode == 0 and not [l for l in out.stdout.splitlines() if l.startswith("{")]


def test_dump_outputs_samples_oversized_states_within_64_mb(tmp_path):
    """dump_outputs with saved states of the fkpp default's size (11 x 256 x 8192 fp32, 92 MB): at most 64 MB in all, headers and
    the trajectory index included; the sample keeps values and float types; two writes give the same files."""
    shape = (11, 256, 8192)
    make = "rng = np.random.default_rng(5); out = rng.standard_normal(%r, dtype=np.float32); grad = rng.standard_normal(311)" % (shape,)
    code = ("import sys, numpy as np; sys.path.insert(0, sys.argv[1]); import bench\n" + make +
            "\nfor d in sys.argv[2:]: bench.dump_outputs(d, {'out': out, 'grad_theta': grad, 'loss': np.ones(1, np.float32)})\n")
    dirs = [tmp_path / "a", tmp_path / "b"]
    subprocess.run([sys.executable, "-c", code, ROOT] + [str(d) for d in dirs], check=True, timeout=300)
    exec(make, globals(), ns := {"np": np})
    names = {"out.npy", "grad_theta.npy", "loss.npy", "out_trajectory_index.npy"}
    for d in dirs:
        assert {f.name for f in d.iterdir()} == names and 0.99 * 64e6 < sum(f.stat().st_size for f in d.iterdir()) <= 64e6
        idx = np.load(d / "out_trajectory_index.npy")
        assert idx.dtype == np.float64 and np.all(np.diff(idx) > 0) and 0 <= idx[0] and idx[-1] < shape[-1]
        got = np.load(d / "out.npy")
        assert got.dtype == np.float32 and got.shape == shape[:-1] + (idx.size,)
        np.testing.assert_array_equal(got, ns["out"][..., idx.astype(np.int64)])
        assert np.array_equal(np.load(d / "grad_theta.npy"), ns["grad"])
    assert all((dirs[0] / n).read_bytes() == (dirs[1] / n).read_bytes() for n in names)
