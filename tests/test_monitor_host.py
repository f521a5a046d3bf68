"""The step monitor's host side without a GPU: combining z-slab plane partials, and the scene's --stats file and
argument."""
import math

import numpy as np
import pytest

from fluidnet_b200 import scene
from fluidnet_b200.monitor import combine_planes


def _partials(nb, gnz, seed=0):
    rs = np.random.RandomState(seed)
    p = rs.rand(nb, gnz, 3)
    p[:, :, 0] *= 1e3
    return p


def test_combine_planes_adds_in_ascending_global_z_whatever_the_split():
    p = _partials(2, 23)
    want = np.empty((2, 3))
    for b in range(2):
        s = 0.0
        for z in range(23):
            s += float(p[b, z, 0])
        want[b] = (math.sqrt(s), p[b, :, 1].max(), p[b, :, 2].max())
    for cuts in ([], [7], [3, 11, 12], list(range(1, 23))):
        edges = [0] + cuts + [23]
        parts = [(a, p[:, a:b]) for a, b in zip(edges[:-1], edges[1:])]
        got = combine_planes(parts[::-1])                   # the ranks' order does not matter
        assert got.tobytes() == want.tobytes(), cuts


def test_combine_planes_refuses_gaps_and_overlaps():
    p = _partials(1, 10)
    with pytest.raises(ValueError, match="missing or given twice"):
        combine_planes([(0, p[:, :4]), (5, p[:, 5:])])
    with pytest.raises(ValueError, match="missing or given twice"):
        combine_planes([(0, p[:, :6]), (5, p[:, 5:])])
    with pytest.raises(ValueError, match="one nb"):
        combine_planes([(0, p[:, :5]), (5, np.zeros((2, 5, 3)))])


def test_stats_file_round_trips_and_refuses_other_files(tmp_path):
    rows = scene.stats_rows([(0, np.array([[1.5, 0.25, 3.0]])), (1, np.array([[0.1 + 0.2, 1e-300, 7.0]]))], 0.1)
    assert rows == [(1, 1.5, 0.25, 3.0 * 0.1), (2, 0.1 + 0.2, 1e-300, 7.0 * 0.1)]
    path = str(tmp_path / "sub" / "stats.csv")
    scene.write_stats(path, rows)
    text = open(path).read().splitlines()
    assert text[0] == "frame,div_norm,div_max,u_max_dt"
    assert text[1].startswith("1,1.5,0.25,")
    assert scene.read_stats(path) == rows                  # every double reads back to the same bits
    other = tmp_path / "other.csv"
    other.write_text("a,b\n1,2\n")
    with pytest.raises(ValueError, match="not a --stats file"):
        scene.read_stats(str(other))


def test_stats_argument_reaches_the_run(monkeypatch):
    seen = []
    monkeypatch.setattr(scene, "run", lambda *a, **k: seen.append((a, k)))
    scene.main(["--res", "32", "--sim-method", "jacobi", "--stats", "out/s.csv"])
    scene.main(["--res", "32", "--sim-method", "jacobi"])
    assert seen[0][1]["stats"] == "out/s.csv"
    assert seen[1][1]["stats"] is None
