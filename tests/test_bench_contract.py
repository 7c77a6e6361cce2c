"""bench.py contract on the CPU: the reference arm (the only arm that runs without a GPU) prints exactly ONE JSON line
on stdout with the keys the driver reads; non-zero ranks of a torchrun launch stay silent; the GPU arm fails loudly
(no JSON, non-zero exit) when there is no CUDA device -- there is no CPU fallback to fall into."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(args, env=None):
    e = dict(os.environ)
    e.update(env or {})
    return subprocess.run([sys.executable, os.path.join(ROOT, "bench.py")] + args, capture_output=True, text=True, cwd=ROOT, env=e, timeout=600)


def test_reference_arm_prints_one_json_line():
    r = _run(["--impl", "reference", "--log-n", "10", "--steps", "2", "--warmup", "1"])
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [l for l in r.stdout.splitlines() if l.strip()]
    assert len(lines) == 1
    d = json.loads(lines[0])
    for k in ("impl", "metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
              "vs_baseline", "dtype", "data", "config", "cpu_baseline", "e2e", "gpu_launches"):
        assert k in d, k
    assert d["impl"] == "reference" and d["unit"] == "GB/s" and d["higher_is_better"] is True and d["vs_baseline"] is None
    assert d["value"] > 0 and d["steps"] == 2 and d["gpu_launches"] == 0
    assert d["cpu_baseline"]["kind"] in ("reference", "port") and d["cpu_baseline"]["cores"] >= 1
    assert d["e2e"]["h2d_bytes_per_step"] == 0 and d["e2e"]["d2h_bytes_per_step"] == 0 and d["e2e"]["value"] == d["value"]


def test_reference_arm_other_ranks_are_silent():
    r = _run(["--impl", "reference", "--gpus", "2", "--log-n", "10", "--steps", "1", "--warmup", "1"], env={"RANK": "1", "WORLD_SIZE": "2", "LOCAL_RANK": "1"})
    assert r.returncode == 0 and r.stdout.strip() == ""


def test_b200_arm_without_a_gpu_fails_loudly():
    import torch
    if torch.cuda.is_available():
        import pytest
        pytest.skip("a GPU is present")
    r = _run(["--steps", "1", "--warmup", "1", "--no-cpu-baseline", "--no-e2e"], env={"CUDA_VISIBLE_DEVICES": ""})
    assert r.returncode != 0
    assert r.stdout.strip() == ""                      # nothing that could be mistaken for a measurement


def test_fill_a_rows_is_the_reference_fill_dealt_cyclically():
    """bench.py fills every rank's shard directly (global block l*G + rank = local row l of data0[i] = i % P, RS.cpp:28-29)."""
    import importlib.util
    import numpy as np
    import torch
    spec = importlib.util.spec_from_file_location("bench_mod", os.path.join(ROOT, "bench.py"))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    N, S, G = 64, 12, 4
    full = (np.arange(N * S, dtype=np.uint64) % bench.P).astype(np.uint32).reshape(N, S)
    for r in range(G):
        got = bench.fill_a_rows(torch, "cpu", r, G, N // G, S).numpy().view(np.uint32)
        assert np.array_equal(got, full[r::G])
    assert bench.GOLDEN_PARITY_HASH_FILL_A[(19, 1024)] == 4272226309       # SURVEY 8c
    class A: log_n = 19; block_bytes = 4096
    assert bench.check_golden(A, 4272226309, "x")["golden_match"] is True
    try:
        bench.check_golden(A, 1, "x")
        assert False, "a wrong hash must abort the run"
    except SystemExit as e:
        assert "PARITY FAILURE" in str(e)
