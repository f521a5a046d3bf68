"""The producer / consumer pipeline of the z-streaming tensor-core convolution (k_conv3_tc_z,
fluidnet_b200/csrc/tfl_cnn_tc.cu) across work items.

A persistent CTA stages the padded planes of all its work items through one ring of three slots, and the slot
hand-over (mbarriers `full` and `empty`) keeps its phase parity per slot across planes and items.  At the automatic
grid most CTAs run one item; the test hook tfl_debug_conv_tc_z_grid caps the grid at 1, 2 and 7 CTAs so that every
CTA runs many items back to back, which is where a wrong parity or a missing release would show.  The capped runs
must reproduce the automatic grid's output bit for bit, every buffer position included (the arithmetic of a voxel
does not depend on which CTA computes it), for layers 1, 2 and 3 in both arithmetic modes.  test_gpu_conv_tc.py and
test_gpu_conv_tc_zstream.py check the automatic grid against float64."""
import ctypes as C

import numpy as np
import pytest

from tc_conv import LAYERS, TY, make_layer, nsm, run_layer, schedule

CAPS = [1, 2, 7]
# (nz, ny, nx), nb, (z_lo, z_hi) or None for all planes
CASES = [
    ((12, 9, 128), 2, None),         # two M tiles per row, ny not a multiple of TY, two batch entries
    ((10, 17, 64), 1, None),         # one M tile per row
    ((9, 13, 61), 2, (1, 8)),        # nx not a multiple of 4, a z range
]


def case_id(c):
    (nz, ny, nx), nb, zr = c
    return "%dx%dx%d-nb%d%s" % (nz, ny, nx, nb, "" if zr is None else "-z%d-%d" % zr)


def _grid_hook():
    from fluidnet_b200 import tfluids
    lib = tfluids.context().lib
    lib.tfl_debug_conv_tc_z_grid.argtypes = [C.c_int]
    return lib


def run_capped(x, w, b, tail, split, z_range, cap):
    lib = _grid_hook()
    assert lib.tfl_debug_conv_tc_z_grid(cap) == 0
    try:
        return run_layer(x, w, b, tail, split, *(z_range or (0, None)))
    finally:
        lib.tfl_debug_conv_tc_z_grid(0)


def check_caps(what, x, w, b, tail, split, z_range):
    ref_out, ref_p = run_capped(x, w, b, tail, split, z_range, 0)
    for cap in CAPS:
        out, p = run_capped(x, w, b, tail, split, z_range, cap)
        for name, got, ref in (("out", out, ref_out), ("p_net", p, ref_p)):
            diff = got.view(np.uint32) != ref.view(np.uint32)
            assert not diff.any(), "%s, grid of %d CTAs: %d values of %s differ from the automatic grid, first at %s" % (
                what, cap, diff.sum(), name, np.argwhere(diff)[0])


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=case_id)
@pytest.mark.parametrize("split", [1, 0], ids=["tf32x3", "tf32"])
@pytest.mark.parametrize("kind", list(LAYERS))
def test_capped_grid_is_bitwise_equal(kind, split, case):
    cin, final = LAYERS[kind]
    shape, nb, z_range = case
    what = "%s %s %s" % (kind, ["tf32", "tf32x3"][split], case_id(case))
    x, w, b, tail = make_layer("scaled", cin, final, shape, nb, 1000 + shape[2] + 7 * split)
    check_caps(what, x, w, b, tail, split, z_range)


@pytest.mark.gpu
@pytest.mark.parametrize("split", [1, 0], ids=["tf32x3", "tf32"])
@pytest.mark.parametrize("kind", list(LAYERS))
def test_capped_grid_z_chunks(kind, split):
    """66 row blocks and z[2, 19): the schedule cuts the range into chunks of several planes, the last one shorter,
    so that consecutive items of a CTA start at different planes."""
    cin, final = LAYERS[kind]
    ny, nz, nx, z_range = 66 * TY[split], 20, 8, (2, 19)
    zc, nzc, _ = schedule(1, ny, nx, *z_range, split, nsm())
    assert nzc > 1 and (z_range[1] - z_range[0]) % zc != 0, (zc, nzc)
    x, w, b, tail = make_layer("signed", cin, final, (nz, ny, nx), 1, 2000 + split)
    check_caps("%s %s z[2, 19) zc %d" % (kind, ["tf32", "tf32x3"][split], zc), x, w, b, tail, split, z_range)
