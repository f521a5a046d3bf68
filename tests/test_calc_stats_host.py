"""calc_stats on the host (no GPU): argument handling, frame loading and grouping, the refusal of mixed shapes, the
evaluation mconf and the CSV round trip."""
import math

import numpy as np
import pytest

from fluidnet_b200 import calc_stats, formats, synth


def _save(path, nx, ny, nz, is3d=True):
    flags = synth.make_flags(nx, ny, nz, is3d)
    U = synth.make_velocity(flags, is3d)
    formats.save_manta_file(str(path), np.zeros_like(flags), U, flags, synth.make_density(flags))
    return str(path)


def test_args():
    a = calc_stats.parse_args(["--synthetic", "7", "--res", "16", "--batch", "3", "--steps", "5"])
    assert (a.synthetic, a.res, a.batch, a.steps, a.frames) == (7, 16, 3, 5, [])
    a = calc_stats.parse_args(["a.bin", "b.bin", "--sim-method", "jacobi"])
    assert a.frames == ["a.bin", "b.bin"] and a.sim_method == "jacobi" and a.steps == 128 and a.batch == 16
    for bad in ([], ["a.bin", "--synthetic", "2"], ["--synthetic", "0"], ["--synthetic", "2", "--batch", "0"],
                ["--synthetic", "2", "--steps", "0"], ["a.bin", "--model", "m", "--synthetic-model"],
                ["a.bin", "--sim-method", "sor"]):
        with pytest.raises(SystemExit):
            calc_stats.parse_args(bad)


def test_grouping_keeps_order_and_a_short_last_batch():
    frames = calc_stats.synthetic_frames(7, 8, 3)
    groups = calc_stats.group(frames, 3)
    assert [(i, [f.source for f in g]) for i, g in groups] == [
        (0, ["synthetic:3", "synthetic:4", "synthetic:5"]), (3, ["synthetic:6", "synthetic:7", "synthetic:8"]),
        (6, ["synthetic:9"])]
    assert [len(g) for _, g in calc_stats.group(frames, 16)] == [7]
    with pytest.raises(ValueError):
        calc_stats.group(frames, 0)


def test_synthetic_frames_are_seeded():
    a, b = calc_stats.synthetic_frames(2, 8, 5), calc_stats.synthetic_frames(2, 8, 5)
    assert np.array_equal(a[1].U, b[1].U) and not np.array_equal(a[0].U, a[1].U)
    assert a[0].shape == (8, 8, 8) and a[0].is3d and not a[0].p.any()
    assert np.array_equal(a[0].flags, a[1].flags)


def test_load_frames_and_refuse_mixed_shapes(tmp_path):
    p1 = _save(tmp_path / "a.bin", 8, 6, 4)
    p2 = _save(tmp_path / "b.bin", 8, 6, 4)
    frames = calc_stats.load_frames([p1, p2])
    assert [f.source for f in frames] == ["a.bin", "b.bin"] and frames[0].shape == (4, 6, 8)
    odd = _save(tmp_path / "odd.bin", 8, 6, 5)
    with pytest.raises(ValueError, match="odd.bin"):
        calc_stats.load_frames([p1, odd])
    flat = _save(tmp_path / "flat.bin", 8, 6, 1, is3d=False)
    with pytest.raises(ValueError, match="flat.bin"):
        calc_stats.load_frames([p1, flat])


def test_eval_mconf():
    m = calc_stats.eval_mconf({"gravityScale": 2.0, "dt": 0.05, "simMethod": "convnet", "maxIter": 100})
    assert m["gravityScale"] == 0 and m["dt"] == 0.05 and m["maxIter"] == 34 and m["simMethod"] == "convnet"
    assert calc_stats.eval_mconf(None, "pcg")["simMethod"] == "pcg"
    assert calc_stats.eval_mconf(None)["advectionMethod"] == "maccormack"
    with pytest.raises(ValueError):
        calc_stats.eval_mconf({"simMethod": "sor"})


def test_csv_round_trip_and_summary(tmp_path):
    rows = [(0, "a.bin", 1, 0.1, 1e-300, 0.3), (0, "a.bin", 2, 1 / 3, float("inf"), 2.5),
            (1, "b.bin", 1, 0.5, 0.25, float("nan")), (1, "b.bin", 2, 2.0, 0.0, 1.0)]
    path = str(tmp_path / "s.csv")
    calc_stats.write_csv(path, rows)
    back = calc_stats.read_csv(path)
    assert [r[:3] for r in back] == [r[:3] for r in rows]
    assert np.array_equal(np.array([r[3:] for r in back]), np.array([r[3:] for r in rows]), equal_nan=True)
    with open(path) as f:
        assert f.readline().strip() == ",".join(calc_stats.COLUMNS)
    lines = []
    means, peak = calc_stats.summarize(rows, 2, lines.append)
    assert means == [0.3, (1 / 3 + 2.0) / 2] and math.isnan(peak) and len(lines) == 2
    with pytest.raises(ValueError):
        calc_stats.write_csv(path, [(0, "a,b", 1, 0.0, 0.0, 0.0)])
    with pytest.raises(ValueError):
        calc_stats.read_csv(_save(tmp_path / "x.bin", 4, 4, 4))
