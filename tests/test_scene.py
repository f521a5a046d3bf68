"""CPU checks of the demo scene (fluidnet_b200/scene.py) and the voxel helpers it places obstacles with
(formats.calculate_bounding_box / pad_voxels_to_dims / flip_diagonal, restating torch/lib/voxel_utils.lua)."""
import struct

import numpy as np
import pytest

from fluidnet_b200 import formats, scene
from fluidnet_b200.tfluids import CellType


def vol(shape, cells, value=1.0):
    v = np.zeros(shape, np.float32)
    for c in cells:
        v[c] = value
    return v


# ---- calculateBoundingBox ------------------------------------------------------------------------------------

def test_bounding_box_is_one_based_and_per_axis():
    v = vol((5, 6, 7), [(1, 2, 3), (3, 4, 3), (2, 2, 5)])
    assert formats.calculate_bounding_box(v) == {"min": [2, 3, 4], "max": [4, 5, 6]}


def test_bounding_box_of_a_single_cell_and_of_negative_slabs():
    assert formats.calculate_bounding_box(vol((1, 1, 1), [(0, 0, 0)])) == {"min": [1, 1, 1], "max": [1, 1, 1]}
    # the reference tests the slab sums, so a slab whose values cancel counts as empty
    v = vol((3, 3, 3), [(1, 1, 1)])
    v[0, 0, 0], v[0, 2, 2] = 1.0, -1.0
    assert formats.calculate_bounding_box(v)["min"][0] == 2


def test_bounding_box_of_an_empty_volume_fails():
    with pytest.raises(Exception):
        formats.calculate_bounding_box(np.zeros((4, 4, 4), np.float32))


# ---- padVoxelsToDims -----------------------------------------------------------------------------------------

def placed(ret):
    idx = np.argwhere(ret != 0)
    return tuple(idx.min(0)), tuple(idx.max(0))


def test_pad_trims_to_the_bounding_box_and_centres():
    v = vol((6, 6, 6), [(1, 2, 3), (2, 3, 3)])           # trimmed: 2 x 2 x 1
    ret = formats.pad_voxels_to_dims(10, 8, 12, v, 0, 0, 0)
    assert ret.shape == (12, 8, 10)
    # floor((12 - 2) / 2) = 5, floor((8 - 2) / 2) = 3, floor((10 - 1) / 2) = 4 (odd padding rounds down)
    assert placed(ret) == ((5, 3, 4), (6, 4, 4))
    assert ret.sum() == v.sum()


def test_pad_with_negative_and_fractional_offsets():
    v = vol((4, 4, 4), [(0, 0, 0), (1, 1, 1)])           # trimmed: 2 x 2 x 2
    # x: floor(4 + 1.5) = 5; y: floor(4 - 0.5) = 3; z: floor(4 - 2.7) = 1
    ret = formats.pad_voxels_to_dims(10, 10, 10, v, 1.5, -0.5, -2.7)
    assert placed(ret) == ((1, 3, 5), (2, 4, 6))
    ret = formats.pad_voxels_to_dims(10, 10, 10, v, 0.99, -0.01, 0)
    assert placed(ret) == ((4, 3, 4), (5, 4, 5))


def test_pad_clamps_the_padding_to_one():
    v = vol((4, 4, 4), [(0, 0, 0), (1, 1, 1)])
    ret = formats.pad_voxels_to_dims(10, 10, 10, v, -100, -4, -3.5)
    assert placed(ret) == ((1, 1, 1), (2, 2, 2))          # max(.., 1): one empty plane before the volume
    # a volume as wide as the grid cannot keep that plane: the paste overruns
    full = np.ones((3, 3, 3), np.float32)
    with pytest.raises(IndexError):
        formats.pad_voxels_to_dims(3, 3, 3, full, 0, 0, 0)


def test_pad_refuses_a_volume_larger_than_the_grid_or_empty():
    with pytest.raises(AssertionError):
        formats.pad_voxels_to_dims(4, 4, 4, np.ones((5, 4, 4), np.float32), 0, 0, 0)
    with pytest.raises(AssertionError):
        formats.pad_voxels_to_dims(4, 4, 4, np.zeros((3, 3, 3), np.float32), 0, 0, 0)
    v = vol((4, 4, 4), [(1, 1, 1)], np.nan)                # the reference's volume-sum check: NaN > 0 is false
    with pytest.raises(AssertionError):
        formats.pad_voxels_to_dims(8, 8, 8, v, 0, 0, 0)


# ---- flipDiagonal --------------------------------------------------------------------------------------------

def reference_flip(v, axis):
    """voxel_utils.lua:238-276 loop for loop (1-based indices, two writes per cell)."""
    d1, d2, d3 = v.shape
    tmp = np.zeros_like(v)
    for i in range(1, d1 + 1):
        for j in range(1, d2 + 1):
            for k in range(1, d3 + 1):
                ii, jj, kk = {0: (i, k, j), 1: (k, j, i), 2: (j, i, k)}[axis]
                tmp[i - 1, j - 1, k - 1] = v[ii - 1, jj - 1, kk - 1]
                tmp[ii - 1, jj - 1, kk - 1] = v[i - 1, j - 1, k - 1]
    return tmp


@pytest.mark.parametrize("axis,shape", [(0, (3, 4, 4)), (1, (4, 3, 4)), (2, (4, 4, 3))])
def test_flip_diagonal_matches_the_reference_loop_in_place(axis, shape):
    v = np.random.default_rng(axis).random(shape).astype(np.float32)
    want = reference_flip(v, axis)
    got = formats.flip_diagonal(v, axis)
    assert got is v
    np.testing.assert_array_equal(v, want)


@pytest.mark.parametrize("axis,shape", [(0, (4, 3, 4)), (1, (4, 4, 3)), (2, (3, 4, 4))])
def test_flip_diagonal_asserts_the_swapped_axes_are_equal(axis, shape):
    with pytest.raises(AssertionError):
        formats.flip_diagonal(np.zeros(shape, np.float32), axis)
    with pytest.raises(AssertionError):
        formats.flip_diagonal(np.zeros((4, 4, 4), np.float32), 3)


# ---- the scene -----------------------------------------------------------------------------------------------

def write_binvox(path, dims, occ_flat):
    """A .binvox file whose run-length body decodes, through the reference parser's quirks (formats.load_binvox), to
    occ_flat: one (value, 1) pair per cell -- a run writes count + 1 = 2 cells and moves on by 1, so the next run
    overwrites the second -- and a final pair the parser drops.  The last cell keeps the value of the one before it
    (the parser stops there), so occ_flat must end with two equal values."""
    assert occ_flat[-1] == occ_flat[-2]
    body = bytearray()
    for v in occ_flat:
        body += bytes([int(v), 1])
    body += bytes([0, 0])
    head = "#binvox 1\ndim %d %d %d\ntranslate 0 0 0\nscale 1\ndata\n" % tuple(dims)
    with open(path, "wb") as f:
        f.write(head.encode("ascii") + bytes(body))


def test_model_res_and_binvox_names():
    assert [scene.model_res(r) for r in (16, 32, 64, 100, 128, 256, 512)] == [8, 16, 32, 32, 64, 128, 256]
    assert scene.binvox_name("arch", 128) == "Y91_arc_64.binvox"
    assert scene.binvox_name("bunny", 64) == "bunny.capped_32.binvox"


def test_empty_domain_matches_the_oracle(orc):
    flags = scene.empty_domain_flags(16)
    want = orc.emptyDomain(np.zeros((1, 1, 16, 16, 16), np.float32), True, 1)
    np.testing.assert_array_equal(flags, want)


def test_scene_flags_from_a_synthetic_binvox_file(tmp_path):
    res, d = 16, 8
    occ = np.zeros((d, d, d), np.uint8)
    occ[2:5, 1:4, 3:7] = 1                                   # file order: the binvox's (dims0, dims1, dims2)
    occ[4, 3, 6] = 0
    path = tmp_path / "Y91_arc_8.binvox"
    write_binvox(path, (d, d, d), occ.reshape(-1))
    assert np.array_equal(formats.load_binvox(str(path))["data"], occ.transpose(0, 2, 1).astype(np.float32))
    # by hand: load (permute 1, 3, 2) then flipDiagonal 2 and 0 reverse the file's axes; trim to the bounding box
    v = occ.transpose(2, 1, 0).astype(np.float32)
    lo, hi = np.argwhere(v).min(0), np.argwhere(v).max(0) + 1
    t = v[lo[0]:hi[0], lo[1]:hi[1], lo[2]:hi[2]]
    assert t.shape == (4, 3, 3)

    def pasted(off_x, off_y, off_z):
        want = np.zeros((res, res, res), np.float32)
        pz = max(int(np.floor((res - t.shape[0]) / 2 + off_z)), 1)
        py = max(int(np.floor((res - t.shape[1]) / 2 + off_y)), 1)
        px = max(int(np.floor((res - t.shape[2]) / 2 + off_x)), 1)
        want[pz:pz + t.shape[0], py:py + t.shape[1], px:px + t.shape[2]] = t
        return want

    for src in (str(path), str(tmp_path)):                   # the file, or the directory holding the demo's name
        vox = scene.obstacle_voxels("arch", res, src)
        np.testing.assert_array_equal(vox, pasted(0, -0.04 * res, 0))
    flags = scene.scene_flags(res, vox)
    inner = flags[0, 0, 1:-1, 1:-1, 1:-1]
    np.testing.assert_array_equal(inner, np.where(vox[1:-1, 1:-1, 1:-1] > 0, np.float32(CellType.TypeObstacle),
                                                  np.float32(CellType.TypeFluid)))
    np.testing.assert_array_equal(flags[0, 0][scene.empty_domain_flags(res)[0, 0] == CellType.TypeObstacle],
                                  np.float32(CellType.TypeObstacle))
    np.testing.assert_array_equal(scene.obstacle_voxels("bunny", res, str(path)), pasted(0.04 * res, 0, 0.04 * res))
    assert scene.obstacle_voxels("plume", res, None) is None
    with pytest.raises(ValueError):
        scene.obstacle_voxels("arch", res, None)


def test_scene_mconf_and_file_names():
    m = scene.scene_mconf(64, "jacobi", {"normalizeInputThreshold": 2e-5, "dt": 0.5, "modelType": "default"})
    assert m["buoyancyScale"] == 1.0 and m["gravityScale"] == 0 and m["dt"] == 0.1
    assert m["maccormackStrength"] == 0.6 and m["maxIter"] == 34 and m["vorticityConfinementAmp"] == 3
    assert m["advectionMethod"] == "maccormackOurs" and m["simMethod"] == "jacobi"
    assert m["normalizeInputThreshold"] == 2e-5 and m["modelType"] == "default"
    assert scene.scene_mconf(128)["buoyancyScale"] == 2.0
    with pytest.raises(ValueError):
        scene.scene_mconf(64, "sor")
    assert scene.density_filename("myModel3D", 0.1) == "density_output_myModel3D_dt0.1.vbox"
    assert scene.density_filename("m", 2.0) == "density_output_m_dt2.vbox"
    assert scene.NUM_FRAMES == 768 and scene.OUTPUT_DECIMATION == 3


def test_density_header_keeps_the_reference_frame_count(tmp_path):
    """The header says numFrames; only every third frame follows it (what the demo's files look like)."""
    p = str(tmp_path / "d.vbox")
    frames = [np.full((2, 3, 4), i, np.float32) for i in range(3)]
    with formats.VboxWriter(p, (4, 3, 2), 9) as w:
        w.write(frames[0])
        w.write_packed(np.ascontiguousarray(frames[1].transpose(2, 1, 0)))
        w.write(frames[2])
    with open(p, "rb") as f:
        assert struct.unpack("<4i", f.read(16)) == (4, 3, 2, 9)
    got = formats.load_vbox(p)
    assert got.shape == (3, 2, 3, 4)
    np.testing.assert_array_equal(got, np.stack(frames))


def test_blender_geometry_zeroes_the_border_planes():
    occ = np.ones((4, 5, 6), np.float32)
    g = scene.blender_geometry(occ)
    assert g[1:-1, 1:-1, 1:-1].all() and g.sum() == 2 * 3 * 4 and occ.all()


def test_scene_refuses_a_resolution_outside_the_demo_range():
    with pytest.raises(ValueError):
        scene.run(res=8, model=object())


def test_lua_shim_defines_the_recorder():
    """fluidnet_b200/lua/tfluids_ffi.lua cannot run here (no LuaJIT): its recorder functions exist and call the five
    entry points (test_abi.py checks the cdef against include/tfl.h)."""
    import os
    import re
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    lua = open(os.path.join(root, "fluidnet_b200", "lua", "tfluids_ffi.lua")).read()
    defined = set(re.findall(r"^function tfluids\.([A-Za-z]+)", lua, flags=re.M))
    for name in ("recorderCreate", "recorderCapture", "recorderTake", "recorderRelease", "recorderDestroy"):
        assert name in defined, name
    for sym in ("create", "capture", "take", "release", "destroy"):
        assert "lib.tfl_recorder_%s(" % sym in lua, sym
