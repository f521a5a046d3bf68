"""Layer-level parity of the tensor-core 3x3x3 convolution (k_conv3_tc, fluidnet_b200/csrc/tfl_cnn_tc.cu).

One layer at a time runs through the test hook tfl_debug_conv3_tc (tfl_api_cnn_debug.cu): the weights are packed by
conv_tc_pack_weights, the activations live in the padded channels-last layout [nb][2 planes][nz+2][py][px][4]
(channels 0-3, 4-7), and the result is compared with torch.nn.functional.conv3d in float64 on the CPU
(padding 1, + bias, ReLU; for the last 3x3x3 layer then the 8->8 1x1x1 layer, ReLU and the 8->1 layer).

Error bound, per output voxel
  S = sum |w| |x| + |b|, evaluated as conv3d(|x|, |w|) + |b| in float64.  The kernel must satisfy
  |gpu - ref| <= kappa * S at every voxel (ReLU is 1-Lipschitz, so the bound on the pre-activation carries over).
  * 3xTF32 (split = 1): a = a_hi + a_lo with a_hi = a truncated to tf32 (exact) and a_lo = a - a_hi (exact in
    fp32, |a_lo| < 2^-10 |a|).  The kernel accumulates hi*hi + hi*lo + lo*hi; wgmma reads the lo operands as
    tf32 again, which loses < 2^-10 |a_lo| < 2^-20 |a| each, and lo*lo (< 2^-20 |a||w|) is dropped: about
    3 * 2^-20 of S from the operands.  The fp32 accumulation path (9 K-steps of the hi*hi accumulator, the
    hi*lo and lo*hi accumulators, their sum, the three x-taps and the bias) is about 20 roundings of at most
    one ulp of a partial sum bounded by S: 20 * 2^-23 = 2^-18.7.  kappa = 2^-16 leaves a factor ~4 over both.
  * TF32 (split = 0): both operands truncated to 10 mantissa bits, 2 * 2^-10 = 2^-9 of S, plus the same
    accumulation: kappa = 2^-8.
  * Final layer: the hidden channels h (error E_h = kappa * S_h) go through the fp32 1x1x1 tail.  In float64:
    E_a = |w4| E_h + g (|w4| (|h| + E_h) + |b4|), then E_p = |w5| E_a + g (|w5| (|a| + E_a) + |b5|), with
    g = 2^-20 (16 ulps, for the eight fused multiply-adds and the shuffle join).  |gpu p - ref p| <= E_p.
test_error_model_emulation (no GPU) replays the operand rounding in numpy and shows that the bound holds for
it and that a 3xTF32 without its lo*hi product fails it; the GPU cases add the accumulation.

Largest err / S measured on an H100 80GB HBM3 (SXM, 700 W power limit) over all the cases below (for the final
layer, err / (E_p / kappa)); each test prints its own:
  3xTF32 (kappa = 2^-16 = 1.53e-5):  layer 1  1.08e-6 (0.07 kappa),  layer 2  8.7e-7 (0.06),  layer 3  6.9e-7 (0.05)
  TF32   (kappa = 2^-8  = 3.91e-3):  layer 1  1.31e-3 (0.34 kappa),  layer 2  1.06e-3 (0.27),  layer 3  7.5e-4 (0.19)
The operand rounding alone, emulated, reaches 0.05 kappa (3xTF32) and 0.36 kappa (TF32) on the 'scaled' inputs, so
wgmma's fp32 accumulation adds little on top; a 3xTF32 without its lo*hi product reaches ~30 kappa on 'nonneg'.

Inputs (all normal floats with full fp32 mantissas; denormals are out of scope): 'signed' uniform values,
'nonneg' activations with non-negative weights (no cancellation: S = |ref|, a dropped or mis-scaled term shows
at full size) and 'scaled' values multiplied per voxel by 2^k, k in [-12, 12] (the hi / lo split across
exponents).  Every batch entry has its own contents.  Layer 1 reads one float4 plane; its unused channel 4-7
plane is filled with NaN and the output must stay finite.

Stray writes: out and p_net start filled with a sentinel; every position outside the valid interior (borders,
pad columns, planes outside [z_lo, z_hi), and all of the buffer a layer kind does not write) must still hold
the sentinel bit for bit, and every interior position must have been written."""
import zlib

import numpy as np
import pytest
import torch

from network_bound import conv_f64
from tc_conv import KAPPA, LAYERS, check_layer, debug_lib, layout, make_layer

INPUTS = ("signed", "nonneg", "scaled")
# (nz, ny, nx), nb: exact tiles and one past / one short of the CTA tile edges of both modes (30 columns,
# TY / TZ = 8 / 6 for TF32, 4 / 5 for 3xTF32), every px - (nx + 2) in 0..3, non-cubic grids, nb > 1.
SHAPES = [((1, 1, 1), 1), ((5, 4, 30), 1), ((6, 8, 30), 1), ((7, 9, 31), 2), ((11, 7, 59), 1),
          ((13, 17, 61), 3), ((24, 3, 88), 1), ((2, 40, 7), 2)]


def tf32(a):
    """Truncation to tf32 (the 10 leading mantissa bits), as the tensor cores read an fp32 operand."""
    return (np.ascontiguousarray(a, np.float32).view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)


def case_id(c):
    (nz, ny, nx), nb = c
    return "%dx%dx%d-nb%d" % (nz, ny, nx, nb)


@pytest.mark.gpu
@pytest.mark.parametrize("case", SHAPES, ids=case_id)
@pytest.mark.parametrize("inputs", INPUTS)
@pytest.mark.parametrize("split", [1, 0], ids=["tf32x3", "tf32"])
@pytest.mark.parametrize("kind", list(LAYERS))
def test_layer_matches_float64(kind, split, inputs, case):
    cin, final = LAYERS[kind]
    shape, nb = case
    what = "%s %s %s %s" % (kind, ["tf32", "tf32x3"][split], inputs, case_id(case))
    x, w, b, tail = make_layer(inputs, cin, final, shape, nb, zlib.crc32(what.encode()))
    check_layer(what, x, w, b, tail, split)


@pytest.mark.gpu
@pytest.mark.parametrize("z_range", [(3, 11), (0, 1), (19, 20)], ids=lambda r: "z%d-%d" % r)
@pytest.mark.parametrize("split", [1, 0], ids=["tf32x3", "tf32"])
@pytest.mark.parametrize("kind", list(LAYERS))
def test_layer_z_range(kind, split, z_range):
    """A launch restricted to output planes [z_lo, z_hi) (what the z-slab driver runs) computes those planes
    from the whole input and leaves every other plane alone."""
    cin, final = LAYERS[kind]
    x, w, b, tail = make_layer("signed", cin, final, (20, 10, 33), 2, 11 + z_range[0])
    check_layer("%s %s z[%d, %d)" % (kind, ["tf32", "tf32x3"][split], *z_range), x, w, b, tail, split, *z_range)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", list(LAYERS))
def test_layer_bench_shape(kind):
    """The bench's 128^3 grid, 3xTF32 (the default mode)."""
    cin, final = LAYERS[kind]
    x, w, b, tail = make_layer("signed", cin, final, (128, 128, 128), 1, 5)
    check_layer("%s tf32x3 128^3" % kind, x, w, b, tail, 1)


@pytest.mark.gpu
def test_layer_hook_rejects_bad_arguments():
    from fluidnet_b200 import tfluids
    from fluidnet_b200._lib import TflError
    lib = debug_lib()
    x, w, b, tail = make_layer("signed", 8, 1, (4, 4, 4), 1, 0)
    px, py = layout(1, 4, 4, 4)
    buf = torch.zeros(1, 2, 6, py, px, 4, device="cuda")
    p = torch.zeros(1, 4, 4, 4, device="cuda")
    ctx = tfluids._ctx_for(buf)
    call = lambda cin, final, z_lo, z_hi: ctx.check(lib.tfl_debug_conv3_tc(
        ctx.h, buf.data_ptr(), buf.data_ptr(), p.data_ptr(), w.ctypes.data, b.ctypes.data, tail.ctypes.data,
        cin, final, 1, 1, 4, 4, 4, z_lo, z_hi))
    for args, msg in (((4, 0, 0, 4), "cin"), ((3, 1, 0, 4), "final"), ((8, 0, -1, 4), "z range"),
                      ((8, 0, 0, 5), "z range"), ((8, 0, 2, 2), "z range")):
        with pytest.raises(TflError, match=msg):
            call(*args)


def emulate(x, w, b, split, drop_lo_hi=False):
    """The kernel's operand rounding in float64 (exact accumulation): TF32 truncates both operands; 3xTF32
    sums hi*hi + hi*lo + lo*hi with the fp32 residual lo truncated to tf32 again."""
    if not split:
        return conv_f64(tf32(x), tf32(w), b)
    xh, wh = tf32(x), tf32(w)
    xl, wl = tf32(x - xh), tf32(w - wh)
    zero = np.zeros_like(b)
    y = conv_f64(xh, wh, b) + conv_f64(xh, wl, zero)
    return y if drop_lo_hi else y + conv_f64(xl, wh, zero)


@pytest.mark.parametrize("inputs", INPUTS)
def test_error_model_emulation(inputs):
    """The per-voxel bound kappa * S is neither vacuous nor too tight for the operand rounding: the emulated
    TF32 and 3xTF32 products stay within it, and dropping the lo*hi product of 3xTF32 breaks it on
    non-negative data (as does single-pass TF32 against the 3xTF32 kappa)."""
    for cin in (3, 8):
        x, w, b, _ = make_layer(inputs, cin, 0, (7, 9, 31), 2, 3)
        ref = conv_f64(x, w, b)
        S = conv_f64(np.abs(x), np.abs(w), np.abs(b))
        for split in (0, 1):
            r = (np.abs(emulate(x, w, b, split) - ref) / S).max()
            assert r <= KAPPA[split], (cin, split, r)
        if inputs == "nonneg":
            assert (np.abs(emulate(x, w, b, 1, drop_lo_hi=True) - ref) / S).max() > 8 * KAPPA[1]
            assert (np.abs(emulate(x, w, b, 0) - ref) / S).max() > 8 * KAPPA[1]
