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
import ctypes as C
import zlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

KAPPA = {1: 2.0 ** -16, 0: 2.0 ** -8}            # split -> per-voxel bound factor
TAIL_ULPS = 2.0 ** -20                            # fp32 rounding of the 1x1x1 tail, relative
SENTINEL = np.float32(12345.0)
LAYERS = {"l1": (3, 0), "l2": (8, 0), "l3": (8, 1)}     # kind -> (cin, final_layer)
INPUTS = ("signed", "nonneg", "scaled")
# (nz, ny, nx), nb: exact tiles and one past / one short of the CTA tile edges of both modes (30 columns,
# TY / TZ = 8 / 6 for TF32, 4 / 5 for 3xTF32), every px - (nx + 2) in 0..3, non-cubic grids, nb > 1.
SHAPES = [((1, 1, 1), 1), ((5, 4, 30), 1), ((6, 8, 30), 1), ((7, 9, 31), 2), ((11, 7, 59), 1),
          ((13, 17, 61), 3), ((24, 3, 88), 1), ((2, 40, 7), 2)]


def tf32(a):
    """Truncation to tf32 (the 10 leading mantissa bits), as the tensor cores read an fp32 operand."""
    return (np.ascontiguousarray(a, np.float32).view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)


def make_layer(inputs, cin, final, shape, nb, seed):
    """x [nb][cin][nz][ny][nx], w [8][cin][3][3][3], b [8], tail [81] (w4[8][8], b4[8], w5[8], b5) or None."""
    rs = np.random.RandomState(seed)
    nz, ny, nx = shape
    bw, bt = 1.0 / np.sqrt(cin * 27), 1.0 / np.sqrt(8)
    lo = 0.0 if inputs == "nonneg" else -1.0
    x = rs.uniform(lo, 1.0, (nb, cin, nz, ny, nx))
    if inputs == "scaled":
        x *= 2.0 ** rs.randint(-12, 13, (nb, 1, nz, ny, nx))
    w = rs.uniform(lo * bw, bw, (8, cin, 3, 3, 3))
    b = rs.uniform(lo * bw, bw, 8)
    tail = rs.uniform(lo * bt, bt, 81) if final else None
    f32 = lambda a: None if a is None else np.ascontiguousarray(a, np.float32)
    return f32(x), f32(w), f32(b), f32(tail)


def conv3d_f64(x, w, b):
    """conv3d(x, w) + b in float64 (padding 1), in z chunks so that the CPU's im2col buffer stays small."""
    xt = F.pad(torch.from_numpy(x).double(), (0, 0, 0, 0, 1, 1))
    wt, bt = torch.from_numpy(w).double(), torch.from_numpy(b).double()
    nz, ny, nx = x.shape[2:]
    step = max(1, (1 << 24) // (ny * nx * w.shape[1] * 27))
    out = [F.conv3d(xt[:, :, z0:min(nz, z0 + step) + 2], wt, bt, padding=(0, 1, 1)) for z0 in range(0, nz, step)]
    return torch.cat(out, dim=2).numpy()


def reference(x, w, b, tail, kappa):
    """(ref, bound): the float64 result of the layer and the per-voxel error bound (module docstring)."""
    pre = conv3d_f64(x, w, b)
    S = conv3d_f64(np.abs(x), np.abs(w), np.abs(b))
    h, Eh = np.maximum(pre, 0.0), kappa * S
    if tail is None:
        return h, Eh
    t = tail.astype(np.float64)
    w4, b4, w5, b5 = t[:64].reshape(8, 8), t[64:72], t[72:80], t[80]
    mix = lambda m, v: np.einsum("oc,bczyx->bozyx", m, v)
    a = np.maximum(mix(w4, h) + b4[:, None, None, None], 0.0)
    Ea = mix(np.abs(w4), Eh) + TAIL_ULPS * (mix(np.abs(w4), np.abs(h) + Eh) + np.abs(b4)[:, None, None, None])
    p = np.einsum("o,bozyx->bzyx", w5, a) + b5
    Ep = (np.einsum("o,bozyx->bzyx", np.abs(w5), Ea)
          + TAIL_ULPS * (np.einsum("o,bozyx->bzyx", np.abs(w5), a + Ea) + abs(b5)))
    return p, Ep


def pack(x, px, py, fill_unused=0.0):
    """[nb][c <= 8][nz][ny][nx] -> padded channels-last [nb][2][nz+2][py][px][4]: zero borders and pad columns.
    Channels >= c are 0, except that a plane holding none of the c channels is `fill_unused`."""
    nb, c, nz, ny, nx = x.shape
    buf = np.zeros((nb, 2, nz + 2, py, px, 4), np.float32)
    for h in range(2):
        if 4 * h >= c:
            buf[:, h] = fill_unused
            continue
        for q in range(min(4, c - 4 * h)):
            buf[:, h, 1:nz + 1, 1:ny + 1, 1:nx + 1, q] = x[:, 4 * h + q]
    return buf


def unpack(buf, nz, ny, nx):
    """Padded channels-last -> [nb][8][nz][ny][nx] (the interior)."""
    inner = buf[:, :, 1:nz + 1, 1:ny + 1, 1:nx + 1, :]               # [nb][2][nz][ny][nx][4]
    return np.ascontiguousarray(np.moveaxis(inner, 5, 2).reshape(buf.shape[0], 8, nz, ny, nx))


def _hook():
    from fluidnet_b200 import tfluids
    lib = tfluids.context().lib
    lib.tfl_debug_conv_tc_layout.argtypes = [C.c_int] * 4 + [C.POINTER(C.c_int32)]
    lib.tfl_debug_conv3_tc.argtypes = [C.c_void_p] * 7 + [C.c_int] * 9
    return lib


def layout(nb, nz, ny, nx):
    out = (C.c_int32 * 2)()
    assert _hook().tfl_debug_conv_tc_layout(nb, nz, ny, nx, out) == 0
    return out[0], out[1]


def run_layer(x, w, b, tail, split, z_lo=0, z_hi=None):
    """One layer on the GPU from sentinel-filled out / p_net.  Returns (out, p_net) as numpy arrays."""
    from fluidnet_b200 import tfluids
    lib = _hook()
    nb, cin, nz, ny, nx = x.shape
    z_hi = nz if z_hi is None else z_hi
    px, py = layout(nb, nz, ny, nx)
    assert px >= nx + 2 and px % 4 == 0 and py == ny + 2
    host_in = pack(x, px, py, fill_unused=np.nan)
    din = torch.from_numpy(host_in).cuda()
    dout = torch.full(host_in.shape, float(SENTINEL), device="cuda")
    dp = torch.full((nb, nz, ny, nx), float(SENTINEL), device="cuda")
    ctx = tfluids._ctx_for(din)
    ptr = lambda a: None if a is None else a.ctypes.data
    ctx.check(lib.tfl_debug_conv3_tc(ctx.h, din.data_ptr(), dout.data_ptr(), dp.data_ptr(), ptr(w), ptr(b), ptr(tail),
                                     cin, 0 if tail is None else 1, split, nb, nz, ny, nx, z_lo, z_hi))
    assert np.array_equal(din.cpu().numpy().view(np.uint32), host_in.view(np.uint32)), "the layer wrote its input"
    return dout.cpu().numpy(), dp.cpu().numpy()


def is_sentinel(a):
    return a.view(np.uint32) == SENTINEL.view(np.uint32)


def check_layer(what, x, w, b, tail, split, z_lo=0, z_hi=None):
    """Run one layer and check it (module docstring).  Returns max err / bound."""
    nb, cin, nz, ny, nx = x.shape
    z_hi = nz if z_hi is None else z_hi
    out, p_net = run_layer(x, w, b, tail, split, z_lo, z_hi)
    ref, bound = reference(x, w, b, tail, KAPPA[split])
    ref, bound = ref[:, :, z_lo:z_hi] if tail is None else ref[:, z_lo:z_hi], \
        bound[:, :, z_lo:z_hi] if tail is None else bound[:, z_lo:z_hi]
    if tail is None:
        assert is_sentinel(p_net).all(), "%s: a hidden layer wrote p_net" % what
        written = np.zeros(out.shape, bool)
        written[:, :, 1 + z_lo:1 + z_hi, 1:ny + 1, 1:nx + 1, :] = True
        stray = ~is_sentinel(out) & ~written
        assert not stray.any(), "%s: %d stray writes in out, first at %s" % (what, stray.sum(), np.argwhere(stray)[0])
        got = unpack(out, nz, ny, nx)[:, :, z_lo:z_hi]
    else:
        assert is_sentinel(out).all(), "%s: the final layer wrote out" % what
        outside = np.ones(p_net.shape, bool)
        outside[:, z_lo:z_hi] = False
        assert is_sentinel(p_net[outside]).all(), "%s: p_net written outside [%d, %d)" % (what, z_lo, z_hi)
        got = p_net[:, z_lo:z_hi]
    missed = is_sentinel(np.ascontiguousarray(got))
    assert not missed.any(), "%s: %d interior values not written, first at %s" % (what, missed.sum(), np.argwhere(missed)[0])
    assert np.isfinite(got).all(), "%s: non-finite output" % what
    err = np.abs(got.astype(np.float64) - ref)
    ratio = err / np.maximum(bound, 1e-300)
    worst = np.unravel_index(np.argmax(ratio), ratio.shape)
    print("conv_tc %s: max err/S %.3e (kappa %.3e)" % (what, ratio.max() * KAPPA[split], KAPPA[split]))
    assert (err <= bound).all(), "%s: %d voxels over the bound; worst %s: err %.3e bound %.3e (ratio %.2f)" % (
        what, (err > bound).sum(), worst, err[worst], bound[worst], ratio[worst])
    return ratio.max()


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
    lib = _hook()
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
        return conv3d_f64(tf32(x), tf32(w), b)
    xh, wh = tf32(x), tf32(w)
    xl, wl = tf32(x - xh), tf32(w - wh)
    zero = np.zeros_like(b)
    y = conv3d_f64(xh, wh, b) + conv3d_f64(xh, wl, zero)
    return y if drop_lo_hi else y + conv3d_f64(xl, wh, zero)


@pytest.mark.parametrize("inputs", INPUTS)
def test_error_model_emulation(inputs):
    """The per-voxel bound kappa * S is neither vacuous nor too tight for the operand rounding: the emulated
    TF32 and 3xTF32 products stay within it, and dropping the lo*hi product of 3xTF32 breaks it on
    non-negative data (as does single-pass TF32 against the 3xTF32 kappa)."""
    for cin in (3, 8):
        x, w, b, _ = make_layer(inputs, cin, 0, (7, 9, 31), 2, 3)
        ref = conv3d_f64(x, w, b)
        S = conv3d_f64(np.abs(x), np.abs(w), np.abs(b))
        for split in (0, 1):
            r = (np.abs(emulate(x, w, b, split) - ref) / S).max()
            assert r <= KAPPA[split], (cin, split, r)
        if inputs == "nonneg":
            assert (np.abs(emulate(x, w, b, 1, drop_lo_hi=True) - ref) / S).max() > 8 * KAPPA[1]
            assert (np.abs(emulate(x, w, b, 0) - ref) / S).max() > 8 * KAPPA[1]
