"""Shared pieces of the fp32 convolution tests: the direct and generic kernel cases, the guarded buffers around a
launch, the activation and its ulp bound, and the quantised inputs."""
import ctypes as C
import zlib

import numpy as np
import torch


SIGMOID_ULPS = 2.0 ** -20


DIRECT, GENERIC = 1, 2                # what tfl_debug_conv_fp32 reports


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


def activate(v, act):
    if act == 1:
        return np.maximum(v, 0.0)
    if act == 2:
        return 1.0 / (1.0 + np.exp(-v))
    return v


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
    lib = debug_lib()
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


def seed_of(what):
    return zlib.crc32(what.encode())


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


U_ROUND = 2.0 ** -24


SENTINEL = 0x7FC0BEEF                 # a NaN payload that no kernel produces from finite inputs


GUARD = 1024                          # floats before and after the output that must keep the sentinel


def debug_lib():
    from fluidnet_b200 import tfluids
    lib = tfluids.context().lib
    lib.tfl_debug_conv_fp32.argtypes = [C.c_void_p] * 5 + [C.c_int] * 10 + [C.POINTER(C.c_int32)]
    lib.tfl_debug_pool.argtypes = [C.c_void_p] * 3 + [C.c_int] * 7
    lib.tfl_debug_pixel_shuffle.argtypes = [C.c_void_p] * 3 + [C.c_int] * 7
    lib.tfl_debug_bank_join.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p] + [C.c_int] * 7
    return lib
