"""Shared pieces of the tensor-core convolution tests: the interleaved TF32 layout and its packing, the layer cases and
their float64 check, the z-streaming schedule, and the join reference."""
import ctypes as C

import numpy as np
import torch

from network_bound import conv_f64


KAPPA = {1: 2.0 ** -16, 0: 2.0 ** -8}            # split -> per-voxel bound factor


TAIL_ULPS = 2.0 ** -20                            # fp32 rounding of the 1x1x1 tail, relative


SENTINEL = np.float32(12345.0)


LAYERS = {"l1": (3, 0), "l2": (8, 0), "l3": (8, 1)}     # kind -> (cin, final_layer)


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


def layout(nb, nz, ny, nx):
    out = (C.c_int32 * 2)()
    assert debug_lib().tfl_debug_conv_tc_layout(nb, nz, ny, nx, out) == 0
    return out[0], out[1]


def run_layer(x, w, b, tail, split, z_lo=0, z_hi=None):
    """One layer on the GPU from sentinel-filled out / p_net.  Returns (out, p_net) as numpy arrays."""
    from fluidnet_b200 import tfluids
    lib = debug_lib()
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
    ref, bound = layer_reference(x, w, b, tail, KAPPA[split])
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


TY = {1: 4, 0: 8}


def schedule(nb, ny, nx, z_lo, z_hi, split, nsm):
    """(zc, nzc, items) of k_conv3_tc_z: ZC minimises rounds x (ZC + 2), ties to the larger ZC."""
    assert nx <= WW_MAX
    cols = nb * -(-ny // TY[split])
    nzo = z_hi - z_lo
    best = None
    for zc in range(1, nzo + 1):
        items = cols * -(-nzo // zc)
        grid = min(items, nsm)
        cost = -(-items // grid) * (zc + 2)
        if best is None or cost <= best[0]:
            best = (cost, zc, -(-nzo // zc), items)
    return best[1:]


def nsm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def join_reference(banks, agg, w, b, tail, kappa):
    ups = [up(x.astype(np.float64), 2 ** i) for i, x in enumerate(banks)]
    if agg == "concat":
        x, xa = np.concatenate(ups, axis=1), np.abs(np.concatenate(ups, axis=1))
    else:
        x, xa = sum(ups[1:], ups[0]), sum((np.abs(u) for u in ups[1:]), np.abs(ups[0]))
    pre = conv_f64(x, w, b)
    S = conv_f64(xa, np.abs(w), np.abs(b))
    h, Eh = np.maximum(pre, 0.0), kappa * S
    t = tail.astype(np.float64)
    w4, b4, w5, b5 = t[:64].reshape(8, 8), t[64:72], t[72:80], t[80]
    mix = lambda m, v: np.einsum("oc,bczyx->bozyx", m, v)
    a = np.maximum(mix(w4, h) + b4[:, None, None, None], 0.0)
    Ea = mix(np.abs(w4), Eh) + TAIL_ULPS * (mix(np.abs(w4), np.abs(h) + Eh) + np.abs(b4)[:, None, None, None])
    p = np.einsum("o,bozyx->bzyx", w5, a) + b5
    Ep = (np.einsum("o,bozyx->bzyx", np.abs(w5), Ea)
          + TAIL_ULPS * (np.einsum("o,bozyx->bzyx", np.abs(w5), a + Ea) + abs(b5)))
    return p, Ep


def layer_reference(x, w, b, tail, kappa):
    """(ref, bound): the float64 result of the layer and the per-voxel error bound (module docstring)."""
    pre = conv_f64(x, w, b)
    S = conv_f64(np.abs(x), np.abs(w), np.abs(b))
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


def debug_lib():
    from fluidnet_b200 import tfluids
    lib = tfluids.context().lib
    lib.tfl_debug_conv_tc_layout.argtypes = [C.c_int] * 4 + [C.POINTER(C.c_int32)]
    lib.tfl_debug_conv3_tc.argtypes = [C.c_void_p] * 7 + [C.c_int] * 9
    return lib


WW_MAX = 128


def up(x, r):
    return np.repeat(np.repeat(np.repeat(x, r, axis=2), r, axis=3), r, axis=4)
