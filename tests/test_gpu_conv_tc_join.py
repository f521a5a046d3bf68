"""Join layer of the banked tensor-core path (k_conv3_tc with the bank loader, fluidnet_b200/csrc/tfl_cnn_tc.cu) on
its own, through the test hook tfl_debug_conv3_tc_join.  Bank i's layer-2 output lives at its own resolution
(grid >> (i-1)) in the padded channels-last layout; the layer must equal, voxel by voxel, the float64
conv3d(cat(b1, up(b2), ...)) ('concat', one launch per bank through an fp32 partial sum) or
conv3d(b1 + up(b2) + ...) ('add', summed while staging), followed by ReLU and the 1x1x1 tail.

Bound: that of tests/test_gpu_conv_tc.py (|err| <= E_p, from kappa * S with S = sum |w| |x| + |b|; kappa = 2^-16 in
3xTF32, 2^-8 in TF32), with |x| for 'add' taken as sum_i |up(b_i)| (the fp32 sum while staging rounds relative to it).
The pad columns of every bank buffer hold NaN, which the loader must never read, and the bank buffers must be left
as they were."""
import ctypes as C
import zlib

import numpy as np
import pytest
import torch

from tc_conv import KAPPA, SENTINEL, is_sentinel, join_reference, layout, pack

pytestmark = pytest.mark.gpu

# (nz, ny, nx) of the full grid, nb, nbanks: coarse nx of 29 / 30 / 31 (one short of, exactly, one past a
# 30-column tile), full nx one short of / exactly / one past two tiles, coarse ny not a multiple of 4 or 8,
# a coarsest bank of 1x1x1, batch of three.
SHAPES = [((10, 8, 60), 1, 2), ((12, 18, 58), 2, 2), ((4, 6, 62), 1, 2), ((8, 20, 120), 1, 3),
          ((4, 4, 4), 2, 3), ((8, 12, 16), 3, 2), ((12, 8, 24), 1, 3)]


def run_join(banks, agg, w, b, tail, split, full):
    from fluidnet_b200 import tfluids
    nz, ny, nx = full
    nb = banks[0].shape[0]
    dev, host = [], []
    for x in banks:
        bz, by, bx = x.shape[2:]
        px, py = layout(nb, bz, by, bx)
        buf = pack(x, px, py)
        buf[:, :, :, :, bx + 2:, :] = np.nan                  # pad columns: never read
        host.append(buf)
        dev.append(torch.from_numpy(buf).cuda())
    p = torch.full((nb, nz, ny, nx), float(SENTINEL), device="cuda")
    ctx = tfluids._ctx_for(p)
    lib = ctx.lib
    lib.tfl_debug_conv3_tc_join.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.c_int, C.c_int, C.c_void_p,
                                            C.c_void_p, C.c_void_p, C.c_void_p] + [C.c_int] * 5
    ptrs = (C.c_void_p * len(dev))(*[d.data_ptr() for d in dev])
    ctx.check(lib.tfl_debug_conv3_tc_join(ctx.h, ptrs, len(dev), 1 if agg == "add" else 0, p.data_ptr(),
                                          w.ctypes.data, b.ctypes.data, tail.ctypes.data, split, nb, nz, ny, nx))
    for d, h in zip(dev, host):
        assert np.array_equal(d.cpu().numpy().view(np.uint32), h.view(np.uint32)), "the join wrote a bank buffer"
    return p.cpu().numpy()


def case_id(c):
    (nz, ny, nx), nb, n = c
    return "%dx%dx%d-nb%d-N%d" % (nz, ny, nx, nb, n)


@pytest.mark.parametrize("case", SHAPES, ids=case_id)
@pytest.mark.parametrize("agg", ["concat", "add"])
@pytest.mark.parametrize("split", [1, 0], ids=["tf32x3", "tf32"])
def test_join_matches_float64(split, agg, case):
    full, nb, n = case
    what = "join %s %s %s" % (["tf32", "tf32x3"][split], agg, case_id(case))
    rs = np.random.RandomState(zlib.crc32(what.encode()))
    nz, ny, nx = full
    banks = [rs.uniform(0.0, 1.0, (nb, 8, nz >> i, ny >> i, nx >> i)).astype(np.float32) for i in range(n)]
    cin = 8 * n if agg == "concat" else 8
    bw, bt = 1.0 / np.sqrt(cin * 27), 1.0 / np.sqrt(8)
    w = rs.uniform(-bw, bw, (8, cin, 3, 3, 3)).astype(np.float32)
    b = rs.uniform(-bw, bw, 8).astype(np.float32)
    tail = rs.uniform(-bt, bt, 81).astype(np.float32)
    got = run_join(banks, agg, w, b, tail, split, full)
    missed = is_sentinel(got)
    assert not missed.any(), "%s: %d voxels not written" % (what, missed.sum())
    assert np.isfinite(got).all(), "%s: non-finite output (a NaN pad column was read)" % what
    ref, bound = join_reference(banks, agg, w, b, tail, KAPPA[split])
    err = np.abs(got.astype(np.float64) - ref)
    ratio = err / np.maximum(bound, 1e-300)
    print("%s: max err / bound %.3f" % (what, ratio.max()))
    assert (err <= bound).all(), "%s: %d voxels over the bound (worst ratio %.2f)" % (what, (err > bound).sum(), ratio.max())


def test_join_hook_rejects_bad_grids():
    from fluidnet_b200 import tfluids
    from fluidnet_b200._lib import TflError
    p = torch.zeros(1, 6, 6, 6, device="cuda")
    ctx = tfluids._ctx_for(p)
    lib = ctx.lib
    lib.tfl_debug_conv3_tc_join.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.c_int, C.c_int, C.c_void_p,
                                            C.c_void_p, C.c_void_p, C.c_void_p] + [C.c_int] * 5
    w = np.zeros(8 * 24 * 27, np.float32)
    ptrs = (C.c_void_p * 3)(p.data_ptr(), p.data_ptr(), p.data_ptr())
    with pytest.raises(TflError, match="divisible"):
        ctx.check(lib.tfl_debug_conv3_tc_join(ctx.h, ptrs, 3, 0, p.data_ptr(), w.ctypes.data, w.ctypes.data,
                                              w.ctypes.data, 1, 1, 6, 6, 6))
