"""Edges of the z-streaming tensor-core convolution (k_conv3_tc_z, fluidnet_b200/csrc/tfl_cnn_tc.cu), checked with
test_gpu_conv_tc.py's float64 reference, per-voxel bound and stray-write checks.

The kernel runs layers 1-3 at nx <= 128 (wider rows keep the one-shot box kernel).  A work item is TY output rows
(3xTF32 4, TF32 8) x the whole row, staged as 64 or 128 positions from padded x = 1, x ZC output planes x one batch
entry, and a persistent grid of one CTA per SM walks the items.  The cases put each of those at an edge: rows that
fill 64 or 128 staged positions exactly or leave them one short, and rows one past 128 (the switch to the box
kernel); row counts one short of and one past a row block; z chunks of more than one plane, whole and with a shorter
last chunk; batch entries in one launch; and more items than CTAs.  `schedule` restates the host's choice
of ZC so that each case can assert the edge it is meant to reach."""
import pytest

from tc_conv import LAYERS, TY, check_layer, make_layer, nsm, schedule

SPLITS = [1, 0]


@pytest.mark.gpu
@pytest.mark.parametrize("nx", [63, 64, 65, 127, 128, 129, 256])
@pytest.mark.parametrize("dy", [-1, 1])
@pytest.mark.parametrize("split", SPLITS, ids=["tf32x3", "tf32"])
@pytest.mark.parametrize("kind", list(LAYERS))
def test_row_window_edges(kind, split, dy, nx):
    """Rows of 63 / 64 / 65 / 127 / 128 positions (one or two M tiles per row, full or one short) and 129 / 256 (the
    box kernel on either side of the switch), with ny one short of / one past a TY-row block, nb = 2."""
    cin, final = LAYERS[kind]
    ny = 2 * TY[split] + dy
    what = "%s %s zstream nx%d ny%d" % (kind, ["tf32", "tf32x3"][split], nx, ny)
    x, w, b, tail = make_layer("scaled", cin, final, (5, ny, nx), 2, nx * 7 + ny)
    check_layer(what, x, w, b, tail, split)


@pytest.mark.gpu
@pytest.mark.parametrize("z_range", [(0, 20), (3, 17), (2, 19), (9, 11), (19, 20)], ids=lambda r: "z%d-%d" % r)
@pytest.mark.parametrize("split", SPLITS, ids=["tf32x3", "tf32"])
@pytest.mark.parametrize("kind", list(LAYERS))
def test_z_chunks(kind, split, z_range):
    """66 row blocks, so that the schedule cuts the z range into chunks of several planes: ranges that are whole
    chunks, one whose last chunk is shorter (z[2, 19): ZC 9 on 132 SMs, 9 + 8 planes), and one- and two-plane
    ranges."""
    cin, final = LAYERS[kind]
    ny, nz, nx = 66 * TY[split], 20, 8
    zc, nzc, _ = schedule(1, ny, nx, *z_range, split, nsm())
    if z_range[1] - z_range[0] > 2:
        assert zc > 1 and nzc > 1, (zc, nzc)
    if z_range == (2, 19):
        assert (z_range[1] - z_range[0]) % zc != 0, zc
    x, w, b, tail = make_layer("signed", cin, final, (nz, ny, nx), 1, 31 + z_range[0])
    check_layer("%s %s zstream z[%d, %d) zc %d" % (kind, ["tf32", "tf32x3"][split], *z_range, zc), x, w, b, tail,
                split, *z_range)


@pytest.mark.gpu
@pytest.mark.parametrize("split", SPLITS, ids=["tf32x3", "tf32"])
@pytest.mark.parametrize("kind", list(LAYERS))
def test_more_items_than_ctas(kind, split):
    """nb = 2 and 70 row blocks per entry: more work items than SMs, so CTAs take several items across batch
    entries."""
    cin, final = LAYERS[kind]
    ny, nz, nx = 70 * TY[split] - 1, 6, 128
    _, _, items = schedule(2, ny, nx, 0, nz, split, nsm())
    assert items > nsm(), items
    x, w, b, tail = make_layer("nonneg", cin, final, (nz, ny, nx), 2, 77)
    check_layer("%s %s zstream items %d" % (kind, ["tf32", "tf32x3"][split], items), x, w, b, tail, split)
