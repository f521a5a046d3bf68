"""Layer-level parity of the fp32 projection-network kernels (fluidnet_b200/csrc/tfl_cnn.cu): the direct convolution
k_conv_direct at every (cout, k) it is specialised for, the generic k_conv_any, k_pool, k_pixel_shuffle and
k_bank_join, one launch at a time through the test hooks tfl_debug_conv_fp32, tfl_debug_pool,
tfl_debug_pixel_shuffle and tfl_debug_bank_join (tfl_api_cnn_debug.cu); and the graph executor (tfl_cnn_forward.cu),
which must keep the entries of a batch apart.

Convolution reference: conv3d in float64 (conv2d for 2-D, as a conv3d with kz = 1), zero padding (k - 1) / 2, plus
the bias, then the activation.  S = conv(|x|, |w|) + |b|, n = cin * taps + 1 terms.

Error bound, per output value
  * Both kernels start from the bias and add one fmaf per in-grid tap, in the order (c, dz, dy, dx): at most n - 1
    roundings of a partial sum, each by at most u = 2^-24 relative.  Summation error analysis gives
    |gpu - ref| <= gamma_n * S with gamma_n = n u / (1 - n u) for the pre-activation; ReLU is 1-Lipschitz and
    carries it over unchanged.
  * Sigmoid, 1 / (1 + expf(-r)): sigma is 1/4-Lipschitz, so an error E on r moves the result by at most E / 4.
    expf is within 2 ulp (CUDA C Programming Guide, without fast math, which the library does not use), and the IEEE
    add and divide round once each: about 4 ulp of sigma relative, bounded here by 2^-20 sigma(ref).  Bound:
    E / 4 + 2^-20 sigma(ref).
Inputs
  * 'exact': x an integer in [-8, 8] times 2^-2, w an integer in [-16, 16] times 2^-4, b an integer in [-64, 64] times
    2^-6.  Every product is a multiple of 2^-6 and every partial sum is below 2^20 of those units (S < 2^14 for every
    case here), so fp32 computes them exactly in any order: E = 0, and with no activation or ReLU the kernel must
    equal float64 as a value (+0 == -0) at any n.  A dropped, repeated or misplaced tap shows at full size.
    test_exact_inputs_are_exact_in_float32 (no GPU) checks this premise against a float32 conv3d on the CPU.
  * 'signed': uniform values with full mantissas, Torch's +-1/sqrt(fan_in) for the weights.
  * 'nonneg': non-negative x and w, so S = |ref| and nothing cancels.
Every case also runs the generic kernel on the same operands (generic = 1): its accumulation order is the direct
kernel's, so the two results must be identical bit for bit.  The output buffer starts as a NaN sentinel with
guards before and after it: the guards must keep it, every output value must be written, and the input must be
left as it was.

pool, pixel shuffle and bank join are exact operations (a sum in a fixed order and one divide, a max, a permutation,
a copy, a float32 sum in bank order): they must equal their float32 emulation bit for bit.

The graph executor: with U quantised to multiples of 2^-8, the double sums behind the input scale are exact in any
order, so the fp32 forward is deterministic voxel by voxel, and entry b of a batch of three must equal, bit for bit,
the forward of entry b alone.  The banked 'concat' graphs run bank 1's last stage one entry at a time with a batch
stride (run_stage's per-entry convolution, pixel shuffle and pooling paths).

Largest err / bound measured on an H100 80GB HBM3 (SXM, 700 W power limit) over all the cases below; each check
prints its own:
  signed   0.52 (no activation or ReLU), 0.16 (sigmoid)
  nonneg   0.54 (no activation or ReLU), 0.14 (sigmoid)
  exact    0 (no activation or ReLU: equal to float64), 0.16 (sigmoid: the 2^-20 sigma term alone)
The largest ratios come from the 1x1 layers (n = 6 terms), where a few roundings in the same direction come close
to gamma_n; the long sums stay far below it.
"""
import ctypes as C
import os
import zlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

U_ROUND = 2.0 ** -24
SIGMOID_ULPS = 2.0 ** -20
SENTINEL = 0x7FC0BEEF                 # a NaN payload that no kernel produces from finite inputs
GUARD = 1024                          # floats before and after the output that must keep the sentinel
DIRECT, GENERIC = 1, 2                # what tfl_debug_conv_fp32 reports
INPUTS = ("exact", "signed", "nonneg")
# The (cout, k) instantiations of k_conv_direct (launch_conv_direct), each in 2-D and 3-D.
INSTANCES = [(8, 3), (8, 1), (1, 1), (16, 3), (16, 1), (1, 3), (6, 3), (6, 1), (32, 1), (16, 5), (32, 5), (64, 5),
             (64, 1)]
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "myModel2D_layers.npz")


def gamma(n):
    return n * U_ROUND / (1.0 - n * U_ROUND)


def make_conv(inputs, cin, cout, k, is3d, shape, nb, seed):
    """x [nb][cin][nz][ny][nx], w [cout][cin][kz][k][k], b [cout] in float32 (module docstring)."""
    rs = np.random.RandomState(seed)
    kz = k if is3d else 1
    xs, ws = (nb, cin) + tuple(shape), (cout, cin, kz, k, k)
    if inputs == "exact":
        x = rs.randint(-8, 9, xs) * 2.0 ** -2
        w = rs.randint(-16, 17, ws) * 2.0 ** -4
        b = rs.randint(-64, 65, cout) * 2.0 ** -6
    else:
        lo = 0.0 if inputs == "nonneg" else -1.0
        bw = 1.0 / np.sqrt(cin * kz * k * k)
        x = rs.uniform(lo, 1.0, xs)
        w = rs.uniform(lo * bw, bw, ws)
        b = rs.uniform(lo * bw, bw, cout)
    return tuple(np.ascontiguousarray(a, np.float32) for a in (x, w, b))


def conv_f64(x, w, b):
    kz, k = w.shape[2], w.shape[4]
    return F.conv3d(torch.from_numpy(x).double(), torch.from_numpy(w).double(), torch.from_numpy(b).double(),
                    padding=((kz - 1) // 2, (k - 1) // 2, (k - 1) // 2)).numpy()


def activate(v, act):
    if act == 1:
        return np.maximum(v, 0.0)
    if act == 2:
        return 1.0 / (1.0 + np.exp(-v))
    return v


def reference(x, w, b, act, exact):
    """(ref, bound): the float64 layer and the per-value error bound of the module docstring."""
    pre = conv_f64(x, w, b)
    S = conv_f64(np.abs(x), np.abs(w), np.abs(b))
    n = int(np.prod(w.shape[1:])) + 1
    E = np.zeros_like(S) if exact else gamma(n) * S
    ref = activate(pre, act)
    return ref, (E / 4 + SIGMOID_ULPS * ref if act == 2 else E)


def _hook():
    from fluidnet_b200 import tfluids
    lib = tfluids.context().lib
    lib.tfl_debug_conv_fp32.argtypes = [C.c_void_p] * 5 + [C.c_int] * 10 + [C.POINTER(C.c_int32)]
    lib.tfl_debug_pool.argtypes = [C.c_void_p] * 3 + [C.c_int] * 7
    lib.tfl_debug_pixel_shuffle.argtypes = [C.c_void_p] * 3 + [C.c_int] * 7
    lib.tfl_debug_bank_join.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p] + [C.c_int] * 7
    return lib


def guarded(n):
    """A device buffer of n floats between two guards, all holding the sentinel: (whole buffer, output view)."""
    buf = torch.full((GUARD + n + GUARD,), SENTINEL, dtype=torch.int32, device="cuda").view(torch.float32)
    return buf, buf[GUARD:GUARD + n]


def check_guards(buf, n, what):
    a = buf.cpu().numpy().view(np.uint32)
    outside = np.concatenate([a[:GUARD], a[GUARD + n:]])
    assert (outside == SENTINEL).all(), "%s: %d stray writes around the output" % (what, (outside != SENTINEL).sum())
    inside = a[GUARD:GUARD + n]
    assert not (inside == SENTINEL).any(), "%s: %d output values not written" % (what, (inside == SENTINEL).sum())
    return inside.view(np.float32)


def run_conv(x, w, b, act, is3d, generic, what):
    """One convolution on the GPU.  Returns (out [nb][cout][nz][ny][nx], the kernel that ran)."""
    from fluidnet_b200 import tfluids
    lib = _hook()
    nb, cin, nz, ny, nx = x.shape
    cout, k = w.shape[0], w.shape[4]
    n = nb * cout * nz * ny * nx
    din = torch.from_numpy(x).cuda()
    buf, out = guarded(n)
    kernel = C.c_int32(0)
    ctx = tfluids._ctx_for(din)
    ctx.check(lib.tfl_debug_conv_fp32(ctx.h, din.data_ptr(), out.data_ptr(), w.ctypes.data, b.ctypes.data, cin, cout,
                                      k, act, int(is3d), nb, nz, ny, nx, generic, C.byref(kernel)))
    assert np.array_equal(din.cpu().numpy().view(np.uint32), x.view(np.uint32)), "%s: wrote its input" % what
    return check_guards(buf, n, what).reshape(nb, cout, nz, ny, nx), kernel.value


def check_conv(what, x, w, b, act, is3d, inputs, kernel, ref=None):
    """Run the layer with the kernel launch_conv_direct picks (which must be `kernel`) and with the generic one;
    check the first against float64 and the second against the first, bit for bit.  Returns the output."""
    got, ran = run_conv(x, w, b, act, is3d, 0, what)
    assert ran == kernel, "%s: ran kernel %d, expected %d" % (what, ran, kernel)
    ref, bound = reference(x, w, b, act, inputs == "exact") if ref is None else ref
    assert np.isfinite(got).all(), "%s: non-finite output" % what
    err = np.abs(got.astype(np.float64) - ref)
    bad = err > bound
    if bad.any():
        worst = np.unravel_index(np.argmax(err - bound), err.shape)
        raise AssertionError("%s: %d values over the bound; worst %s: gpu %r ref %r bound %.3e" % (
            what, bad.sum(), worst, got[worst], ref[worst], bound[worst]))
    ratio = (err / np.where(bound > 0, bound, 1.0)).max()
    print("conv_fp32 %s %s act%d: max err/bound %.3e" % (inputs, what, act, ratio))
    gen, ran = run_conv(x, w, b, act, is3d, 1, what + " generic")
    assert ran == GENERIC
    diff = gen.view(np.uint32) != got.view(np.uint32)
    assert not diff.any(), "%s: generic and direct differ at %d values, first %s" % (what, diff.sum(), np.argwhere(diff)[0])
    return got


def seed_of(what):
    return zlib.crc32(what.encode())


@pytest.mark.gpu
@pytest.mark.parametrize("act", [0, 1, 2], ids=["none", "relu", "sigmoid"])
@pytest.mark.parametrize("is3d", [True, False], ids=["3d", "2d"])
@pytest.mark.parametrize("inst", INSTANCES, ids=lambda i: "c%dk%d" % i)
def test_every_direct_instantiation(inst, is3d, act):
    """All 26 (cout, k, 2-D / 3-D) instantiations of k_conv_direct.  nz = 5 with nb = 2: a z pair of threads of the
    3-D block straddles the two entries."""
    cout, k = inst
    shape, nb, cin = ((5, 6, 37) if is3d else (1, 11, 37)), 2, 5
    for inputs in INPUTS:
        what = "c%dk%d %s" % (cout, k, "3d" if is3d else "2d")
        x, w, b = make_conv(inputs, cin, cout, k, is3d, shape, nb, seed_of(what + inputs + str(act)))
        check_conv(what, x, w, b, act, is3d, inputs, DIRECT)


# Shapes outside the specialised table: 2-D 'tog''s last layer (4 = 1 x 2^2 channels before the pixel shuffle),
# 3-D 'tog''s 256-channel 1x1x1 layer, and cout 8 with k 5.
GENERIC_SHAPES = [(4, 3, False, 16), (256, 1, True, 32), (8, 5, True, 3), (8, 5, False, 3)]


@pytest.mark.gpu
@pytest.mark.parametrize("act", [0, 1, 2], ids=["none", "relu", "sigmoid"])
@pytest.mark.parametrize("case", GENERIC_SHAPES, ids=lambda c: "c%dk%d-%s" % (c[0], c[1], "3d" if c[2] else "2d"))
def test_generic_shapes(case, act):
    cout, k, is3d, cin = case
    shape = (3, 7, 33) if is3d else (1, 9, 33)
    for inputs in INPUTS:
        what = "generic c%dk%d %s" % (cout, k, "3d" if is3d else "2d")
        x, w, b = make_conv(inputs, cin, cout, k, is3d, shape, 2, seed_of(what + inputs + str(act)))
        check_conv(what, x, w, b, act, is3d, inputs, GENERIC)


# Grids at the edges of k_conv_direct's blocks, (32, 4, 2) in 3-D and (32, 8, 1) in 2-D: nx one short of, at and
# one past a block row, two rows; ny across the block's 4 / 8; nz and nb such that nb * nz is odd (a z pair of
# threads straddles two entries, or its second thread is past the last one); grids smaller than the kernel.
EDGES_3D = [((1, 1, 1), 1), ((1, 1, 1), 3), ((2, 3, 31), 1), ((3, 4, 32), 1), ((3, 5, 33), 3), ((1, 4, 70), 3),
            ((2, 5, 70), 2), ((3, 3, 1), 2), ((1, 5, 32), 1), ((3, 1, 33), 3), ((2, 4, 31), 3), ((1, 3, 33), 2)]
EDGES_2D = [((1, 7, 1), 1), ((1, 8, 31), 3), ((1, 9, 33), 2), ((1, 7, 32), 3), ((1, 8, 70), 1), ((1, 9, 1), 3),
            ((1, 1, 1), 2)]


@pytest.mark.gpu
@pytest.mark.parametrize("inst", [(8, 3), (64, 5), (1, 1), (16, 5)], ids=lambda i: "c%dk%d" % i)
@pytest.mark.parametrize("case", EDGES_3D, ids=lambda c: "%dx%dx%d-nb%d" % (c[0] + (c[1],)))
def test_grid_edges_3d(case, inst):
    shape, nb = case
    cout, k = inst
    for inputs in ("exact", "signed"):
        what = "edge c%dk%d 3d %s nb%d" % (cout, k, shape, nb)
        x, w, b = make_conv(inputs, 3, cout, k, True, shape, nb, seed_of(what + inputs))
        check_conv(what, x, w, b, 1, True, inputs, DIRECT)


@pytest.mark.gpu
@pytest.mark.parametrize("inst", [(16, 3), (32, 5), (1, 1), (8, 3)], ids=lambda i: "c%dk%d" % i)
@pytest.mark.parametrize("case", EDGES_2D, ids=lambda c: "%dx%d-nb%d" % (c[0][1:] + (c[1],)))
def test_grid_edges_2d(case, inst):
    shape, nb = case
    cout, k = inst
    for inputs in ("exact", "signed"):
        what = "edge c%dk%d 2d %s nb%d" % (cout, k, shape, nb)
        x, w, b = make_conv(inputs, 3, cout, k, False, shape, nb, seed_of(what + inputs))
        check_conv(what, x, w, b, 1, False, inputs, DIRECT)


# One channel on each side of conv_launch's two switch points in shared memory (cin * taps * cout floats):
# at or below 48 KiB no attribute is needed, above it the kernel's attribute is raised (and cached per
# instantiation and device), above 200 KiB the generic kernel runs.
SMEM = {
    "2d-c32k5": (False, 32, 5, (1, 9, 33), [15, 16, 64, 65]),
    "3d-c8k3": (True, 8, 3, (3, 5, 33), [56, 57, 237, 238]),
    "3d-c64k5": (True, 64, 5, (3, 4, 9), [1, 2, 6, 7]),
}


def smem_bytes(is3d, cout, k, cin):
    return 4 * cin * (k if is3d else 1) * k * k * cout


def test_smem_table_sits_on_the_limits():
    """The channel counts of SMEM straddle 48 KiB and 200 KiB as their names say."""
    for is3d, cout, k, _, cins in SMEM.values():
        a, b, c, d = (smem_bytes(is3d, cout, k, cin) for cin in cins)
        assert a <= 48 * 1024 < b and c <= 200 * 1024 < d


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(SMEM))
def test_shared_memory_switch_points(name):
    """Largest first, then smallest first: the attribute raised for a large cin must serve a smaller one, and a
    larger one must raise it again."""
    is3d, cout, k, shape, cins = SMEM[name]
    refs = {}
    for order in (cins[::-1], cins):
        for cin in order:
            kernel = GENERIC if smem_bytes(is3d, cout, k, cin) > 200 * 1024 else DIRECT
            for inputs in INPUTS:
                what = "smem %s cin%d" % (name, cin)
                x, w, b = make_conv(inputs, cin, cout, k, is3d, shape, 2, seed_of(what + inputs))
                key = (cin, inputs)
                if key not in refs:
                    refs[key] = reference(x, w, b, 1, inputs == "exact")
                check_conv(what, x, w, b, 1, is3d, inputs, kernel, refs[key])


@pytest.mark.gpu
def test_shipped_model_layer_by_layer():
    """The trained 2-D model the reference ships, one layer at a time on a 64^2 grid: layer l reads the GPU's output
    of layer l - 1, so each layer is checked on its own (no compounding).  Input: a zero pDiv channel, a smooth
    divergence and the occupancy of a grid with geometry, as the network sees them."""
    from fluidnet_b200 import synth
    z = np.load(GOLD)
    n_layers = int(z["n_layers"])
    n = 64
    flags = synth.make_flags(n, n, 1, False, nb=1, geometry=True)
    rs = np.random.RandomState(3)
    x = np.zeros((1, 3, 1, n, n), np.float32)
    x[:, 1] = rs.uniform(-1.0, 1.0, (1, 1, n, n))
    x[:, 2] = (flags[:, 0] != synth.FLUID).astype(np.float32)
    for l in range(n_layers):
        w, b = np.ascontiguousarray(z["w%d" % l], np.float32), np.ascontiguousarray(z["b%d" % l], np.float32)
        act = 1 if l < n_layers - 1 else 0
        x = np.ascontiguousarray(check_conv("myModel2D layer %d" % (l + 1), x, w, b, act, False, "signed", DIRECT))


@pytest.mark.gpu
def test_conv_hook_rejects_bad_arguments():
    from fluidnet_b200 import tfluids
    from fluidnet_b200._lib import TflError
    lib = _hook()
    x, w, b = make_conv("signed", 3, 8, 3, True, (2, 2, 2), 1, 0)
    d = torch.zeros(64, device="cuda")
    ctx = tfluids._ctx_for(d)
    kernel = C.c_int32(0)
    call = lambda k, act, is3d, nz, generic: ctx.check(lib.tfl_debug_conv_fp32(
        ctx.h, d.data_ptr(), d.data_ptr(), w.ctypes.data, b.ctypes.data, 3, 8, k, act, is3d, 1, nz, 2, 2, generic,
        C.byref(kernel)))
    for args, msg in (((2, 0, 1, 2, 0), "bad layer"), ((3, 3, 1, 2, 0), "bad layer"), ((3, 0, 1, 2, 2), "bad layer"),
                      ((3, 0, 0, 2, 0), "bad grid"), ((3, 0, 1, 0, 0), "bad grid")):
        with pytest.raises(TflError, match=msg):
            call(*args)


def test_exact_inputs_are_exact_in_float32():
    """The premise of the 'exact' class: at the largest n of this file, a float32 conv3d on the CPU (its own
    summation order) equals float64, and every partial sum stays below 2^20 units of 2^-6."""
    for cin, cout, k, is3d in ((238, 8, 3, True), (65, 32, 5, False), (7, 64, 5, True), (32, 256, 1, True)):
        shape = (3, 5, 9) if is3d else (1, 9, 11)
        x, w, b = make_conv("exact", cin, cout, k, is3d, shape, 2, cin)
        pad = ((w.shape[2] - 1) // 2, (k - 1) // 2, (k - 1) // 2)
        f32 = F.conv3d(torch.from_numpy(x), torch.from_numpy(w), torch.from_numpy(b), padding=pad).numpy()
        assert np.array_equal(f32.astype(np.float64), conv_f64(x, w, b))
        S = conv_f64(np.abs(x), np.abs(w), np.abs(b))
        assert S.max() * 64 < 2 ** 20


# ---------------------------------------------------------------------------------------------------------------
# pooling, pixel shuffle, bank join: bit for bit
# ---------------------------------------------------------------------------------------------------------------

def pool_emulation(x, p, is3d, is_max):
    """k_pool in float32: the window in (dz, dy, dx) order from 0 (avg, then / float32(count)) or -inf (max)."""
    nbc, nz, ny, nx = x.shape
    pz = p if is3d else 1
    v = x.reshape(nbc, nz // pz, pz, ny // p, p, nx // p, p)
    acc = np.full((nbc, nz // pz, ny // p, nx // p), -np.inf if is_max else 0.0, np.float32)
    for dz in range(pz):
        for dy in range(p):
            for dx in range(p):
                t = v[:, :, dz, :, dy, :, dx]
                acc = np.maximum(acc, t) if is_max else (acc + t).astype(np.float32)
    return acc if is_max else acc / np.float32(pz * p * p)


@pytest.mark.gpu
@pytest.mark.parametrize("nbc", [1, 5, 48])
@pytest.mark.parametrize("is3d", [True, False], ids=["3d", "2d"])
@pytest.mark.parametrize("p", [2, 3])
@pytest.mark.parametrize("kind", ["avg", "max"])
def test_pool_bit_exact(kind, p, is3d, nbc):
    from fluidnet_b200 import tfluids
    lib = _hook()
    nz, ny, nx = (3 * p if is3d else 1), 5 * p, 7 * p
    x = np.random.RandomState(seed_of("pool%s%d%d%d" % (kind, p, is3d, nbc))).standard_normal(
        (nbc, nz, ny, nx)).astype(np.float32)
    want = pool_emulation(x, p, is3d, kind == "max")
    din = torch.from_numpy(x).cuda()
    buf, out = guarded(want.size)
    ctx = tfluids._ctx_for(din)
    ctx.check(lib.tfl_debug_pool(ctx.h, din.data_ptr(), out.data_ptr(), nbc, nz, ny, nx, p, int(is3d),
                                 int(kind == "max")))
    got = check_guards(buf, want.size, "pool").reshape(want.shape)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), "%d values differ" % (got != want).sum()
    assert np.array_equal(din.cpu().numpy(), x)


def shuffle_reference(x, n_out, s, is3d):
    """The view / permute of ConvolutionUpsample: channel ((o sT + st) s + sh) s + sw -> (o, z sT + st, y s + sh,
    x s + sw)."""
    nb, _, nz, ny, nx = x.shape
    st = s if is3d else 1
    t = torch.from_numpy(x).view(nb, n_out, st, s, s, nz, ny, nx).permute(0, 1, 5, 2, 6, 3, 7, 4)
    return np.ascontiguousarray(t.reshape(nb, n_out, nz * st, ny * s, nx * s).numpy())


@pytest.mark.gpu
@pytest.mark.parametrize("n_out", [1, 4, 32])
@pytest.mark.parametrize("nb", [1, 3])
@pytest.mark.parametrize("is3d", [True, False], ids=["3d", "2d"])
@pytest.mark.parametrize("s", [2, 3])
def test_pixel_shuffle_bit_exact(s, is3d, nb, n_out):
    from fluidnet_b200 import tfluids
    lib = _hook()
    st = s if is3d else 1
    nz, ny, nx = (3 if is3d else 1), 5, 7
    x = np.random.RandomState(seed_of("shuffle%d%d%d%d" % (s, is3d, nb, n_out))).standard_normal(
        (nb, n_out * st * s * s, nz, ny, nx)).astype(np.float32)
    want = shuffle_reference(x, n_out, s, is3d)
    din = torch.from_numpy(x).cuda()
    buf, out = guarded(want.size)
    ctx = tfluids._ctx_for(din)
    ctx.check(lib.tfl_debug_pixel_shuffle(ctx.h, din.data_ptr(), out.data_ptr(), nb, n_out, nz, ny, nx, s, int(is3d)))
    got = check_guards(buf, want.size, "pixel shuffle").reshape(want.shape)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


def upsample(x, r, is3d):
    y = np.repeat(np.repeat(x, r, axis=3), r, axis=4)
    return np.repeat(y, r, axis=2) if is3d else y


def join_grid(nbanks, is3d):
    r = 1 << (nbanks - 1)
    if is3d:
        return 2 * r, 3 * r, 5 * r
    return (1, 3 * r, 5 * r) if r <= 16 else (1, r, 2 * r)


def run_join(bank_list, agg, out_init, is3d, nbanks=None):
    from fluidnet_b200 import tfluids
    lib = _hook()
    nbanks = len(bank_list) if nbanks is None else nbanks
    nb, c = bank_list[0].shape[:2]
    nz, ny, nx = bank_list[0].shape[2:]
    dev = [torch.from_numpy(x).cuda() for x in bank_list]
    ptrs = (C.c_void_p * max(nbanks, len(dev)))(*([None] + [d.data_ptr() for d in dev[1:]]))
    buf, out = guarded(out_init.size)
    out.copy_(torch.from_numpy(out_init.reshape(-1)))
    ctx = tfluids._ctx_for(out)
    ctx.check(lib.tfl_debug_bank_join(ctx.h, ptrs, nbanks, out.data_ptr(), nb, c, nz, ny, nx, int(is3d),
                                      int(agg == "add")))
    for d, x in zip(dev, bank_list):
        assert np.array_equal(d.cpu().numpy().view(np.uint32), x.view(np.uint32)), "the join wrote a bank"
    a = buf.cpu().numpy().view(np.uint32)
    assert (a[:GUARD] == SENTINEL).all() and (a[GUARD + out_init.size:] == SENTINEL).all(), "stray writes"
    return a[GUARD:GUARD + out_init.size].view(np.float32).reshape(out_init.shape)


JOINS = [(True, 2), (True, 3), (True, 4), (False, 2), (False, 5), (False, 8)]     # 8 = kMaxBankPtrs


@pytest.mark.gpu
@pytest.mark.parametrize("nb", [1, 3])
@pytest.mark.parametrize("c", [1, 8, 32])
@pytest.mark.parametrize("case", JOINS, ids=lambda j: "%s-n%d" % ("3d" if j[0] else "2d", j[1]))
@pytest.mark.parametrize("agg", ["concat", "add"])
def test_bank_join_bit_exact(agg, case, c, nb):
    """'concat': channel block i of bank 1's tensor becomes bank i upsampled nearest, block 1 is left alone; 'add':
    bank 1 plus the upsampled banks 2..N, summed in bank order in float32."""
    is3d, nbanks = case
    nz, ny, nx = join_grid(nbanks, is3d)
    rs = np.random.RandomState(seed_of("join%s%d%d%d%d" % (agg, is3d, nbanks, c, nb)))
    banks = []
    for i in range(nbanks):
        shape = (nb, c, nz >> i if is3d else nz, ny >> i, nx >> i)
        banks.append(rs.standard_normal(shape).astype(np.float32))
    ups = [banks[0]] + [upsample(banks[i], 1 << i, is3d) for i in range(1, nbanks)]
    if agg == "concat":
        init = np.full((nb, nbanks * c, nz, ny, nx), np.nan, np.float32)
        init[:, :c] = banks[0]
        want = np.concatenate(ups, axis=1)
    else:
        init = banks[0].copy()
        want = banks[0].copy()
        for u in ups[1:]:
            want = (want + u).astype(np.float32)
    got = run_join(banks, agg, init, is3d)
    diff = got.view(np.uint32) != want.view(np.uint32)
    assert not diff.any(), "%d values differ, first at %s" % (diff.sum(), np.argwhere(diff)[0])


@pytest.mark.gpu
@pytest.mark.parametrize("nbanks", [1, 9])
def test_bank_join_refuses_bank_counts(nbanks):
    from fluidnet_b200._lib import TflError
    banks = [np.zeros((1, 1, 1, 256, 256), np.float32) for _ in range(min(nbanks, 8))]
    with pytest.raises(TflError, match="bank count"):
        run_join(banks, "add", banks[0], False, nbanks=nbanks)


# ---------------------------------------------------------------------------------------------------------------
# the graph executor keeps batch entries apart
# ---------------------------------------------------------------------------------------------------------------

def banks(num, agg, s=1, j=3):
    return {"num": num, "split_stage": s, "join_stage": j, "aggregate": agg}


# (is3d, model_type, poolType, banks, (nz, ny, nx)); every model runs in fp32 mode.
GRAPHS = {
    "2d-default": (False, "default", "avg", None, (1, 20, 24)),
    "3d-default": (True, "default", "avg", None, (6, 10, 12)),
    "2d-tog-avg": (False, "tog", "avg", None, (1, 20, 24)),
    "2d-tog-max": (False, "tog", "max", None, (1, 20, 24)),
    "3d-tog-avg": (True, "tog", "avg", None, (8, 12, 16)),
    "3d-tog-max": (True, "tog", "max", None, (8, 12, 16)),
    "2d-yang": (False, "yang", "avg", None, (1, 20, 24)),
    "3d-yang": (True, "yang", "avg", None, (6, 10, 12)),
    "3d-default-n2-concat": (True, "default", "avg", banks(2, "concat"), (8, 12, 16)),
    "3d-default-n3-add": (True, "default", "avg", banks(3, "add"), (8, 12, 16)),
    "3d-default-n2-concat-s2j4": (True, "default", "avg", banks(2, "concat", 2, 4), (6, 10, 12)),
    "3d-default-n2-add-s2j4": (True, "default", "avg", banks(2, "add", 2, 4), (6, 10, 12)),
    "3d-yang-n2-add-s1j2": (True, "yang", "avg", banks(2, "add", 1, 2), (6, 8, 10)),
    "3d-yang-n2-concat-s1j2": (True, "yang", "avg", banks(2, "concat", 1, 2), (6, 8, 10)),
    "2d-default-n3-concat": (False, "default", "avg", banks(3, "concat"), (1, 24, 20)),
    "2d-tog-n2-concat": (False, "tog", "avg", banks(2, "concat"), (1, 32, 48)),
    "2d-tog-n2-add": (False, "tog", "max", banks(2, "add"), (1, 32, 48)),
    # bank 1's last stage pools (split 1, join 2) / pixel-shuffles (shuffle_model) one entry at a time
    "2d-tog-n2-concat-s1j2": (False, "tog", "avg", banks(2, "concat", 1, 2), (1, 32, 48)),
    "3d-shuffle-n2-concat-s2j3": (True, "shuffle", "avg", banks(2, "concat", 2, 3), (8, 12, 16)),
    "2d-shuffle-n3-concat-s2j3": (False, "shuffle", "max", banks(3, "concat", 2, 3), (1, 24, 32)),
}


def shuffle_model(is3d, nbanks, seed=4321):
    """A graph whose last banked stage ends in a pixel shuffle (no stock graph has one before its join): 3 -> 8 (k 3,
    pool 2), 8 -> 8 (k 1, up 2; one per bank), 8 nbanks -> 8 (k 3, the 'concat' join), 8 -> 1 (k 1)."""
    rs = np.random.RandomState(seed)
    kz = lambda k: k if is3d else 1
    fan = 8 if is3d else 4

    def conv(cout, cin, k):
        bound = 1.0 / np.sqrt(cin * kz(k) * k * k)
        w = ((rs.rand(cout, cin, kz(k), k, k) * 2 - 1) * bound).astype(np.float32)
        return w, ((rs.rand(cout) * 2 - 1) * bound).astype(np.float32)

    layers = [conv(8, 3, 3), [conv(8 * fan, 8, 1) for _ in range(nbanks)], conv(8, 8 * nbanks, 3), conv(1, 8, 1)]
    return {"is3D": is3d, "layers": layers, "pool": [2, 1, 1, 1], "up": [1, 2, 1, 1]}


def quantised_batch(shape, is3d, nb, seed):
    """flags with Empty / Outflow / Stick cells that differ per entry, U and pDiv on multiples of 2^-8."""
    from fluidnet_b200 import synth
    nz, ny, nx = shape
    flags = synth.make_flags(nx, ny, nz, is3d, nb=nb, geometry=True, exotic=True, seed=seed)
    U = synth.make_smooth_velocity(flags, is3d, amp=3.0, seed=seed)
    p = synth.make_density(flags, seed=seed + 1) - np.float32(0.5)
    q = lambda a: np.ascontiguousarray(np.round(a * 256.0) / 256.0, np.float32)
    return q(p), q(U), flags


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(GRAPHS))
def test_batch_entries_are_independent(name):
    """Entry b of a batch of three equals, bit for bit, the forward of entry b alone (p and U)."""
    from fluidnet_b200 import synth
    from fluidnet_b200 import model as fmodel
    is3d, model_type, pool_type, bk, shape = GRAPHS[name]
    if model_type == "shuffle":
        mnp = shuffle_model(is3d, bk["num"])
    else:
        mnp = synth.make_model(is3d, model_type=model_type, banks=bk)
    gm = fmodel.ProjectionModel(mnp["layers"], is3d, pool=mnp.get("pool"), up=mnp.get("up"), poolType=pool_type,
                                nonlinType=mnp.get("nonlinType", "relu"), banks=bk)
    gm.set_mode("fp32")
    arrays = quantised_batch(shape, is3d, 3, seed_of(name) % 10000)
    p3, U3 = gm.forward(tuple(torch.from_numpy(a).cuda() for a in arrays))
    p3, U3 = p3.cpu().numpy(), U3.cpu().numpy()
    assert np.isfinite(p3).all() and np.abs(p3).max() > 0
    for b in range(3):
        one = tuple(torch.from_numpy(np.ascontiguousarray(a[b:b + 1])).cuda() for a in arrays)
        p1, U1 = (t.cpu().numpy() for t in gm.forward(one))
        for got, want, k in ((p3[b:b + 1], p1, "p"), (U3[b:b + 1], U1, "U")):
            diff = got.view(np.uint32) != want.view(np.uint32)
            assert not diff.any(), "%s: entry %d of the batch: %s differs from its own forward at %d voxels, first %s" % (
                name, b, k, diff.sum(), np.argwhere(diff)[0])
