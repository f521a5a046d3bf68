"""bench.py pieces that can be checked without a GPU: the synthetic problem of the measured arm is built
by the product's own host code (no oracle on that path) and equals what the oracle's builder gives, and
the reference arm prints the contract's JSON line, and --dump-outputs writes what it promises."""
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_problem_inputs_match_oracle_builder():
    sys.path.insert(0, ROOT)
    import bench
    from oracle.api import create_plume_bcs
    batch, mconf, model = bench.make_problem(32)
    ref = {k: batch[k].copy() for k in ("pDiv", "UDiv", "flags", "density")}
    create_plume_bcs(ref, [1.0], 32 / 128.0, 0.15)
    for k in ("UBC", "UBCInvMask", "densityBC", "densityBCInvMask"):
        assert np.array_equal(batch[k], ref[k]), k
    assert mconf["simMethod"] == "convnet" and model["is3D"] is True


def test_reference_arm_json_line():
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--grid", "32",
                          "--steps", "1", "--warmup", "0"], capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-2000:]
    line = [l for l in out.stdout.splitlines() if l.startswith("{")][-1]
    d = json.loads(line)
    for key in ("impl", "metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better",
                "scaling", "vs_baseline", "dtype", "data", "config", "cpu_baseline", "e2e"):
        assert key in d, key
    assert d["impl"] == "reference" and d["value"] > 0 and d["e2e"]["h2d_bytes_per_step"] == 0
    assert d["cpu_baseline"]["kind"] in ("reference", "port")


def test_dump_outputs_writes_float32_within_the_limit(tmp_path, monkeypatch):
    """--dump-outputs: whole fields under the limit; above it, the same seeded sample of each field every run."""
    import torch
    sys.path.insert(0, ROOT)
    import bench
    f = {"p": torch.arange(1000, dtype=torch.float32).reshape(1, 1, 10, 10, 10), "U": torch.ones(1, 3, 10, 10, 10)}
    bench.dump_outputs(str(tmp_path / "whole"), f)
    p = np.load(tmp_path / "whole" / "p.npy")
    assert p.dtype == np.float32 and p.shape == (1, 1, 10, 10, 10) and np.array_equal(p.ravel(), np.arange(1000))
    monkeypatch.setattr(bench, "DUMP_LIMIT_BYTES", 4000)
    for d in ("a", "b"):
        bench.dump_outputs(str(tmp_path / d), f)
    total = sum(os.path.getsize(os.path.join(tmp_path, "a", n)) - 128 for n in os.listdir(tmp_path / "a"))
    assert total <= 4000
    for n in ("p", "p_index", "U", "U_index"):
        assert np.array_equal(np.load(tmp_path / "a" / (n + ".npy")), np.load(tmp_path / "b" / (n + ".npy")))
    idx = np.load(tmp_path / "a" / "p_index.npy")
    assert idx.dtype == np.float64 and np.array_equal(np.load(tmp_path / "a" / "p.npy"), idx.astype(np.float32))
