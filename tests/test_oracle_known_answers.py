"""Data-free known-answer tests the reference itself holds for this path, run against the
oracle (and, when built, the compiled reference):
  * emptyDomain / flagsToOccupancy  -- torch/tfluids/test_tfluids.lua:675-753
  * line-trace geometry             -- torch/tfluids/generic/CalcLineTraceTest.m:24-151
plus the committed golden fixtures generated from the compiled reference
(tests/golden/make_golden.py)."""
import os

import numpy as np
import pytest

import oracle
import ref_record
from cases import bits_equal, describe_diff

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def backends():
    return [oracle.Oracle(), ref_record.reference()]


@pytest.mark.parametrize("be", backends(), ids=lambda b: b.name)
def test_empty_domain(be):
    # test_tfluids.lua:675-708: border cells are TypeObstacle, the rest TypeFluid.
    for is3d in (False, True):
        for bnd in (1, 2, 3):
            nz = 9 if is3d else 1
            f = np.full((2, 1, nz, 10, 11), 77, np.float32)
            be.emptyDomain(f, is3d, bnd)
            for b in range(2):
                for k in range(nz):
                    for j in range(10):
                        for i in range(11):
                            border = (i < bnd or i > 11 - 1 - bnd or j < bnd or j > 10 - 1 - bnd or
                                      (is3d and (k < bnd or k > nz - 1 - bnd)))
                            assert f[b, 0, k, j, i] == (2 if border else 1)


@pytest.mark.parametrize("be", backends(), ids=lambda b: b.name)
def test_flags_to_occupancy(be):
    # test_tfluids.lua:710-753: fluid -> 0, obstacle -> 1, anything else is an error.
    rs = np.random.RandomState(3)
    f = np.where(rs.rand(2, 1, 5, 6, 7) < 0.5, 1.0, 2.0).astype(np.float32)
    occ = be.flagsToOccupancy(f)
    assert np.array_equal(occ, (f == 2).astype(np.float32))
    f[0, 0, 1, 2, 3] = 4.0
    with pytest.raises(RuntimeError):
        be.flagsToOccupancy(f)


def _flags_from_obstacles(obs_xyz):
    """obs[x][y][z] (MATLAB order) -> flags [1][1][z][y][x]; empty cells are fluid."""
    o = np.transpose(obs_xyz, (2, 1, 0))
    return np.ascontiguousarray(np.where(o, 2.0, 1.0).astype(np.float32)[None, None])


@pytest.mark.parametrize("be", backends(), ids=lambda b: b.name)
def test_line_trace_single_voxel(be):
    # CalcLineTraceTest.m:24-58: from every free cell centre towards one occupied voxel.
    dims = (3, 4, 5)
    obs = np.zeros(dims, bool)
    obs[1, 2, 3] = True
    flags = _flags_from_obstacles(obs)
    filled = np.array([1.5, 2.5, 3.5])
    count = 0
    for z in range(dims[2]):
        for y in range(dims[1]):
            for x in range(dims[0]):
                pos = np.array([x, y, z]) + 0.5
                if np.linalg.norm(filled - pos) <= 1e-5:
                    continue
                delta = 0.9 * (filled - pos) - np.array([0.001, 0, 0])
                hit, new_pos = be.calcLineTrace(pos, delta, flags)
                assert hit, (pos, delta)
                # never inside the occupied voxel, never outside the domain
                assert not (1 <= new_pos[0] <= 2 and 2 <= new_pos[1] <= 3 and 3 <= new_pos[2] <= 4)
                assert np.all(new_pos > 0) and np.all(new_pos < np.array(dims))
                count += 1
    assert count == 59


def _sphere_scene():
    width, height, depth = 26, 33, 28
    u, v, z = np.meshgrid(np.arange(1, width + 1), np.arange(1, height + 1), np.arange(1, depth + 1),
                          indexing="ij")
    ctr = (width / 2, height / 2, depth / 2)
    rad = min(width, depth, height) / 4 + 0.5
    obs = ((u - ctr[0]) ** 2 + (v - ctr[1]) ** 2 + (z - ctr[2]) ** 2) <= rad * rad
    return (width, height, depth), _flags_from_obstacles(obs)


@pytest.mark.parametrize("be", backends(), ids=lambda b: b.name)
def test_line_trace_borders_and_corners(be):
    # CalcLineTraceTest.m:101-151.
    dims, flags = _sphere_scene()
    dimsf = np.array(dims, np.float64)
    for dim in range(3):                      # positive faces
        pos = dimsf / 2
        pos[dim] = dims[dim] - 4.1
        delta = np.zeros(3)
        delta[dim] = 6.1
        expected = pos.copy()
        expected[dim] = dims[dim]
        hit, new_pos = be.calcLineTrace(pos, delta, flags)
        assert hit and np.linalg.norm(new_pos - expected) < 1e-4
    for dim in range(3):                      # negative faces
        pos = dimsf / 2
        pos[dim] = 4.1
        delta = np.zeros(3)
        delta[dim] = -6.1
        expected = pos.copy()
        expected[dim] = 0
        hit, new_pos = be.calcLineTrace(pos, delta, flags)
        assert hit and np.linalg.norm(new_pos - expected) < 1e-4
    rs = np.random.RandomState(11)            # case 3: off all borders
    pos = np.array([dims[0] - 5.2, dims[1] - 6.3, dims[2] - 7.4])
    delta = rs.rand(3) * 10 + 10
    hit, new_pos = be.calcLineTrace(pos, delta, flags)
    assert hit
    assert (abs(new_pos[0] - dims[0]) < 1e-4 or abs(new_pos[1] - dims[1]) < 1e-4 or
            abs(new_pos[2] - dims[2]) < 1e-4)
    pos = np.array([dims[0] - 1.5, dims[1] - 1.5, dims[2] - 1.5])      # case 4: exact corner
    hit, new_pos = be.calcLineTrace(pos, np.array([2.0, 2.0, 2.0]), flags)
    assert hit and np.linalg.norm(new_pos - dimsf) < 1e-4
    pos = np.array([dims[0] - 0.5, 0.5, dims[2] - 0.5])                # mixed corner
    hit, new_pos = be.calcLineTrace(pos, np.array([2.0, -2.0, 2.0]), flags)
    assert hit and np.linalg.norm(new_pos - np.array([dims[0], 0, dims[2]])) < 1e-4
    pos = np.array([5.5, dims[1] - 3.2, 11.1])                         # case 5: hits the sphere
    hit, _ = be.calcLineTrace(pos, dimsf / 3 - pos, flags)
    assert hit


def test_no_displacement_is_not_traced(orc):
    # generic/vec3.h:119-127 + calc_line_trace.cc:334-339: |delta|^2 <= 1e-6 -> no step.
    _, flags = _sphere_scene()
    hit, new_pos = orc.calcLineTrace([3.5, 3.5, 3.5], [9e-4, 0, 0], flags)
    assert not hit and np.array_equal(new_pos, np.array([3.5, 3.5, 3.5], np.float32))


def _golden_files():
    if not os.path.isdir(GOLD):
        return []
    return sorted(f for f in os.listdir(GOLD) if f.startswith("ref_") and f.endswith(".npz"))


@pytest.mark.parametrize("fname", _golden_files())
def test_oracle_matches_golden(orc, fname):
    """Fixtures were produced by the compiled reference (tests/golden/make_golden.py)."""
    from golden_util import replay
    z = np.load(os.path.join(GOLD, fname))
    for key, got, want in replay(orc, z):
        assert bits_equal(got, want), "%s %s: %s" % (fname, key, describe_diff(got, want))
