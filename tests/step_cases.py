"""Shared pieces of the fused-step tests: the path cases and their batches, the per-mode and operator-sequence
tolerances, the library contexts of one test, the kernel names one step ran, and the launch tally against the
profiler."""
import ctypes as C
import json
import os
import subprocess
import sys
import warnings
from collections import Counter

import numpy as np
import pytest
import torch

import oracle
from fluidnet_b200 import synth


# conv arithmetic -> tolerance relative to max|field| (tf32 = single-pass TF32 tensor cores, 10-bit mantissa inputs,
# is the "fast" mode and not the default)
MODE_TOL = {"fp32": 2e-5, "tf32x3": 2e-5, "tf32": 3e-3}


OPS_TOL = 1e-6


def case(shape, nb=1, flags="geom", state="plume", method="maccormackOurs", tile=None, amp=3.0, mode="tf32x3",
         pbc=False, threshold=1e-5, **mconf):
    """shape = (nz, ny, nx); flags: geom (sphere + slab) | empty | open (fluid on the x and z faces) | exotic;
    state: plume | none (no density, no BCs) | density (no BCs) | ubc (density + velocity BC) |
    ubc-nodens (velocity BC, no density) | random (random U and density BCs, -0.0 in U and the BCs) |
    unaligned (plume on 4-byte aligned views); tile: tfl_debug_advect_tile mode (None: automatic);
    amp: velocity amplitude (traces of amp * dt cells); mconf: overrides of BASE_MCONF."""
    m = oracle.default_mconf(**BASE_MCONF)
    m.update(mconf)
    m["advectionMethod"] = method
    m["normalizeInputThreshold"] = threshold
    return dict(shape=shape, nb=nb, flags=flags, state=state, method=method, tile=tile, amp=amp, mode=mode,
                pbc=pbc, threshold=threshold, mconf=m)


def takes_fused_path(c):
    """fused_step_applies (tfl_api.cu) for the 3-D convnet steps these tests run with the default input block: a
    tensor-core mode and no pressure BC, at any nb."""
    return c["mode"] != "fp32" and not c["pbc"]


def quad_dims(nb, nz, ny, nx):
    """(grid, block) of the 4-voxel kernels, or None where the per-voxel kernels run."""
    if nx % 4 != 0:
        return None
    quads = nx // 4
    if quads >= 32:
        bx = 32
    elif quads & (quads - 1) == 0:
        bx = quads
    else:
        return None
    bz = 2 if nz > 1 else 1
    by = 256 // (bx * bz)
    return ((quads + bx - 1) // bx, (ny + by - 1) // by, (nb * nz + bz - 1) // bz), (bx, by, bz)


def plume_bcs(batch, nb):
    """createPlumeBCs per batch entry, each with its own velocity, density and radius."""
    parts = []
    for b in range(nb):
        sub = {"UDiv": batch["UDiv"][b:b + 1], "density": batch["density"][b:b + 1]}
        nx = sub["UDiv"].shape[-1]
        oracle.create_plume_bcs(sub, [1.0 - 0.3 * b], nx / 128.0 * 4 * (1 + b), 0.15 + 0.05 * b)
        parts.append(sub)
    for k in ("UBC", "UBCInvMask", "densityBC", "densityBCInvMask"):
        batch[k] = np.ascontiguousarray(np.concatenate([p[k] for p in parts]))


def make_batch(orc, c, seed=1234):
    flags = make_flags(c)
    U = synth.make_smooth_velocity(flags, True, amp=c["amp"], seed=seed)
    orc.setWallBcsForward(U, flags)
    batch = {"pDiv": ((synth.make_density(flags, seed=seed + 1) - np.float32(0.5)) * np.float32(0.1)),
             "UDiv": U, "flags": flags}
    state = c["state"]
    if state != "none" and state != "ubc-nodens":
        batch["density"] = synth.make_density(flags, seed=seed + 2)
    if state in ("plume", "unaligned"):
        plume_bcs(batch, c["nb"])
    elif state in ("ubc", "ubc-nodens"):
        tmp = {"UDiv": U, "density": np.zeros_like(flags)}
        plume_bcs(tmp, c["nb"])
        batch["UBC"], batch["UBCInvMask"] = tmp["UBC"], tmp["UBCInvMask"]
    elif state == "random":
        random_bcs(batch, seed + 3)
        rs = np.random.RandomState(seed + 4)
        U[rs.rand(*U.shape) < 0.05] = -0.0
    if c["pbc"]:
        inv = np.ones_like(flags)
        inv[:, :, 2:5, 3:7, 4:9] = 0.0
        batch["pBCInvMask"] = inv
        batch["pBC"] = np.where(inv == 0, np.float32(0.05), np.float32(0.0)).astype(np.float32)
    return {k: np.ascontiguousarray(v, np.float32) for k, v in batch.items()}


def close_per_entry(got, want, tol, what):
    for b in range(got.shape[0]):
        err = np.abs(got[b].astype(np.float64) - want[b].astype(np.float64)).max()
        scale = max(float(np.abs(want[b]).max()), 1e-6)
        assert err <= tol * scale, "%s[%d]: max err %g vs scale %g (tol %g)" % (what, b, err, scale, tol)


def same_zero_bits(got, want):
    z = (got == 0) | (want == 0)
    return np.array_equal(got[z].view(np.uint32), want[z].view(np.uint32))


def step_path(kernels):
    """'quad', 'scalar' (the fused step's 4-voxel or per-voxel kernels) or 'ops' (neither: the operator sequence),
    from the names of the kernels one step ran."""
    names = list(kernels)
    quad = any("k_cnn_finish_fused4" in k for k in names)
    scalar = any("k_cnn_finish_fused" in k and "k_cnn_finish_fused4" not in k for k in names)
    assert not (quad and scalar), names
    if quad or scalar:
        assert any("k_vort_bc_mask" in k for k in names), names
        return "quad" if quad else "scalar"
    assert not any("k_vort_bc_mask" in k for k in names), names
    return "ops"


def run_in_child(module, expr, timeout=900):
    """json.loads of what `expr` (evaluated after `import <module> as t`) returns in a fresh interpreter.  The profiler
    runs there: on one H100 run, a profiler session opened in the test process left every capture of
    test_gpu_launch_tally.py, later in the same process, without a kernel event."""
    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ)
    env["PYTHONPATH"] = os.pathsep.join(p for p in (here, os.path.dirname(here), env.get("PYTHONPATH")) if p)
    code = "import json, %s as t; print(json.dumps(%s))" % (module, expr)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env, timeout=timeout)
    assert r.returncode == 0, r.stderr[-4000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


class Contexts:
    """Library contexts of one test, each with its own arena (where the step keeps the BC quad mask), flag cache
    (byte flags and clearance) and tile telemetry.  `use(ctx)` makes one the context tfluids calls through, `model`
    creates a model on it.  close() puts back the context tfluids used before, destroys the models, then the
    contexts (a model is destroyed through the context it was created on)."""

    def __init__(self):
        from fluidnet_b200 import tfluids
        self.tfluids = tfluids
        self.dev = torch.cuda.current_device()
        self.saved = tfluids._contexts.get(self.dev)
        self.made, self.models = [], []

    def new(self):
        ctx = self.tfluids.Context(self.dev)
        self.made.append(ctx)
        return ctx

    def use(self, ctx):
        self.tfluids._contexts[self.dev] = ctx

    def model(self, ctx, mnp):
        from fluidnet_b200.model import ProjectionModel
        self.use(ctx)
        m = ProjectionModel.from_model(mnp)
        assert m.ctx is ctx
        self.models.append(m)
        return m

    def close(self):
        torch.cuda.synchronize()
        if self.saved is None:
            self.tfluids._contexts.pop(self.dev, None)
        else:
            self.tfluids._contexts[self.dev] = self.saved
        for m in self.models:
            if m.h:
                m.ctx.lib.tfl_cnn_destroy(m.ctx.h, m.h)
                m.h = None
        for ctx in self.made:
            ctx.lib.tfl_destroy(ctx.h)
            ctx.h = None


@pytest.fixture
def contexts():
    cs = Contexts()
    try:
        yield cs
    finally:
        cs.close()


def run(what, plane, fn, *arrays):
    """fn(*views) on guarded device copies of `arrays`; returns (host copies of the views, fn's value, launches)."""
    gd = Guards(plane)
    views = [gd.put(a) for a in arrays]
    c = ctx()
    c.trace_faults()
    l0 = c.launch_count()
    ret = fn(*views)
    torch.cuda.synchronize()
    launches = c.launch_count() - l0
    gd.check(what)
    assert c.trace_faults() == 0, "%s: trace faults" % what
    return [v.cpu().numpy() for v in views], ret, launches


def set_tile_mode(mode):
    c = ctx()
    c.lib.tfl_debug_advect_tile.argtypes = [C.c_void_p, C.c_int]
    assert c.lib.tfl_debug_advect_tile(c.h, -1 if mode is None else mode) == 0


def plane_of(fl):
    return fl.shape[-1] * fl.shape[-2]


def fill(shape, v=123.0):
    return np.full(shape, v, np.float32)


def profiled_kernels(fn):
    """Counter of the kernels (memcpy and memset left out) the profiler saw while fn ran."""
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return Counter(ev.name for ev in prof.events()
                   if ev.device_type == torch.autograd.DeviceType.CUDA
                   and not ev.name.startswith(("Memcpy", "Memset")))


def tally_and_kernels(ctx, call, attempts=3):
    """(what `call` added to ctx's launch tally, Counter of the kernels the profiler saw it run).

    The profiler can lose a whole capture: on one H100 run it reported no kernel at all for a step that had enqueued
    20.  So every capture brackets the call with two marker kernels of known names (one torch add each), and a capture
    that misses a marker proves nothing about the call: it is taken again, and after `attempts` such captures the
    test fails.  The markers are removed from the count exactly; everything else the capture saw is the call's."""
    call()
    torch.cuda.synchronize()
    buf = torch.zeros(1, device="cuda")
    mark = lambda: buf.add_(1.0)
    lost = 0
    for _ in range(attempts):
        marks = profiled_kernels(lambda: (mark(), mark()))
        if sum(marks.values()) != 2:
            lost += 1
            continue
        before = ctx.launch_count()
        seen = profiled_kernels(lambda: (mark(), call(), mark()))
        tally = ctx.launch_count() - before
        if all(seen[k] >= n for k, n in marks.items()):
            if lost:
                warnings.warn("the profiler lost %d capture(s) before this one" % lost)
            return tally, seen - marks
        lost += 1
    raise AssertionError("the profiler lost its marker kernels in %d captures out of %d" % (lost, attempts))


BASE_MCONF = dict(dt=0.1, maccormackStrength=0.6, buoyancyScale=0.5, vorticityConfinementAmp=3.0,
                  simMethod="convnet")


def make_flags(c):
    nz, ny, nx = c["shape"]
    kind = c["flags"]
    f = synth.make_flags(nx, ny, nz, True, nb=c["nb"], geometry=kind != "empty", exotic=kind == "exotic")
    if kind == "open":           # fluid on the x and z faces (the y faces stay solid)
        f[:, :, :, 1:-1, 0] = synth.FLUID
        f[:, :, :, 1:-1, -1] = synth.FLUID
        f[:, :, 0, 1:-1, :] = synth.FLUID
        f[:, :, -1, 1:-1, :] = synth.FLUID
    return np.ascontiguousarray(f)


def random_bcs(batch, seed, density=True):
    """BC arrays that are the identity pair (invMask 1, bc +0.0) on some quads (4 cells along x) only.  Other
    quads hold invMask 1 with bc -0.0 (not the identity: x + -0.0 keeps a -0.0), or invMask in {0, 0.5, 1} with
    values, zeros and -0.0.  The density BC is additive where invMask is 1 and bc != 0."""
    rs = np.random.RandomState(seed)
    U = batch["UDiv"]
    nb, nc, nz, ny, nx = U.shape
    nq = (nx + 3) // 4

    def per_quad(a):
        return np.ascontiguousarray(np.repeat(a, 4, axis=-1)[..., :nx])

    def arrays(nch, scale):
        kind = per_quad(rs.randint(0, 4, size=(nb, 1, nz, ny, nq)))
        kind = np.broadcast_to(kind, (nb, nch, nz, ny, nx))
        inv = np.where(kind <= 1, 1.0, rs.choice([0.0, 0.5, 1.0], size=kind.shape)).astype(np.float32)
        val = (rs.randn(*kind.shape) * scale).astype(np.float32)
        r = rs.rand(*kind.shape)
        val[r < 0.3] = 0.0
        val[(r >= 0.3) & (r < 0.5)] = -0.0
        bc = np.where(kind == 0, np.float32(0.0), np.where(kind == 1, np.float32(-0.0), val)).astype(np.float32)
        return np.ascontiguousarray(bc), np.ascontiguousarray(inv)

    batch["UBC"], batch["UBCInvMask"] = arrays(nc, 0.5)
    if density:
        dbc, dinv = arrays(1, 0.25)
        batch["densityBC"], batch["densityBCInvMask"] = np.where(dbc == 0, dbc, np.abs(dbc)), dinv   # +0 / -0 kept


class Guards:
    """Device views of host arrays, each inside its own buffer with `g` sentinel words on either side."""

    def __init__(self, plane):
        self.g = (max(plane, 64) + 3) // 4 * 4
        self.bufs = []

    def put(self, a):
        a = np.ascontiguousarray(a, np.float32)
        buf = torch.empty(2 * self.g + a.size, dtype=torch.float32, device="cuda")
        buf.view(torch.int32).fill_(SENTINEL)
        v = buf[self.g:self.g + a.size].view(a.shape)
        v.copy_(torch.from_numpy(a))
        assert v.data_ptr() % 16 == 0 and v.is_contiguous()
        self.bufs.append((buf, a.size))
        return v

    def check(self, what):
        for i, (buf, n) in enumerate(self.bufs):
            bits = buf.view(torch.int32)
            assert bool((bits[:self.g] == SENTINEL).all()), "%s: array %d written before its start" % (what, i)
            assert bool((bits[self.g + n:] == SENTINEL).all()), "%s: array %d written past its end" % (what, i)


SENTINEL = 0x7FC5A5A5          # a quiet NaN with a payload


def ctx():
    from fluidnet_b200 import tfluids
    return tfluids.context()
