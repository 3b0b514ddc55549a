"""CPU suite: the parts of bench.py's contract that do not need a GPU -- the reference arm's JSON line and the refusal of the
product arm to run (or fall back) without a device."""
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(*args, timeout=600):
    return subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), *args], capture_output=True, text=True, timeout=timeout, cwd=ROOT)


def test_reference_arm_prints_the_contract_line():
    r = _run("--impl", "reference", "--steps", "1", "--warmup", "0", "--genes", "400", "--samples", "24", "--cpu-sample-genes", "200")
    assert r.returncode == 0, r.stderr[-2000:]
    line = json.loads(r.stdout.strip().splitlines()[-1])
    assert line["impl"] == "reference" and line["unit"] == "genes/s" and line["higher_is_better"] is True
    assert line["metric"].startswith("genes/sec") and line["value"] > 0 and line["steps"] == 1 and line["n_gpus"] == 1
    assert line["cpu_baseline"]["kind"] == "port" and line["cpu_baseline"]["cores"] >= 1 and line["cpu_baseline"]["value"] == line["value"]
    assert line["e2e"] == {"value": line["value"], "unit": "genes/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    assert "workload" in line["config"] and line["scaling"] == "weak" and line["dtype"] == "f64"


def test_reference_arm_runs_exactly_the_requested_steps():
    r = _run("--impl", "reference", "--steps", "7", "--warmup", "2", "--genes", "300", "--samples", "12", "--cpu-sample-genes", "100")
    assert r.returncode == 0, r.stderr[-2000:]
    line = json.loads(r.stdout.strip().splitlines()[-1])
    assert line["steps"] == 7 and line["warmup"] == 2 and len(line["cpu_baseline"]["pass_s"]) == 7


def test_dump_outputs_is_refused_for_the_reference_arm(tmp_path):
    r = _run("--impl", "reference", "--steps", "1", "--dump-outputs", str(tmp_path / "d"))
    assert r.returncode != 0 and "--dump-outputs" in r.stderr and not (tmp_path / "d").exists()


def _bench_module():
    import importlib.util

    spec = importlib.util.spec_from_file_location("bench_under_test", os.path.join(ROOT, "bench.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _fake_result(G, p=2):
    from types import SimpleNamespace

    rng = np.random.default_rng(1)
    res = {k: rng.random(G) for k in ("dispersions", "genewise", "map", "pvalue", "stat", "se", "normed_means")}
    res.update(lfc=rng.random((G, p)), lfc_converged=np.ones(G), trend=SimpleNamespace(coeffs=np.array([0.1, 2.0])),
               prior_var=0.25, squared_logres=0.5)
    return res


def test_dump_outputs_writes_every_array_below_the_cap(tmp_path):
    bench = _bench_module()
    res = _fake_result(500)
    bench.dump_outputs(str(tmp_path), res)
    assert not (tmp_path / "gene_index.npy").exists()
    for k in ("dispersions", "lfc", "lfc_converged", "trend_coeffs", "prior_var"):
        got = np.load(tmp_path / f"{k}.npy")
        assert got.dtype == np.float64
    np.testing.assert_array_equal(np.load(tmp_path / "lfc.npy"), res["lfc"])
    assert float(np.load(tmp_path / "prior_var.npy")) == 0.25


def test_dump_outputs_samples_genes_above_the_cap(tmp_path):
    bench = _bench_module()
    res, cap = _fake_result(20000), 200_000
    for d in ("a", "b"):
        bench.dump_outputs(str(tmp_path / d), res, cap=cap)
    files = sorted(os.listdir(tmp_path / "a"))
    assert sum(os.path.getsize(tmp_path / "a" / f) for f in files) <= cap
    idx = np.load(tmp_path / "a" / "gene_index.npy").astype(np.int64)
    assert 1000 < len(idx) < 20000 and np.all(np.diff(idx) > 0)
    np.testing.assert_array_equal(np.load(tmp_path / "a" / "lfc.npy"), res["lfc"][idx])
    np.testing.assert_array_equal(np.load(tmp_path / "a" / "pvalue.npy"), res["pvalue"][idx])
    for f in files:  # the sample is fixed: the same genes every time
        np.testing.assert_array_equal(np.load(tmp_path / "a" / f), np.load(tmp_path / "b" / f))


def test_product_arm_fails_loudly_without_a_gpu():
    import ctypes

    try:  # with a visible CUDA device the product arm runs: nothing to check here
        if ctypes.CDLL("libcuda.so.1").cuInit(0) == 0:
            n = ctypes.c_int(0)
            ctypes.CDLL("libcuda.so.1").cuDeviceGetCount(ctypes.byref(n))
            if n.value > 0:
                return
    except OSError:
        pass
    r = _run("--steps", "1", "--warmup", "1", "--genes", "200", "--samples", "12", "--no-cpu-baseline")
    assert r.returncode != 0
    assert "no CPU fallback" in r.stderr and not r.stdout.strip().startswith("{")
