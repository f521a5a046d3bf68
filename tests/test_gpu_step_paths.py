"""The whole step (tfl_simulate_step) on every path it dispatches, and its CUDA-graph form under state changes.

Every row of CASES runs three steps three ways from one state:
  * tfl_simulate_step (simulate.simulate_fused): the fused kernels of tfl_fused.cu (4-voxel quad kernels or the
    per-voxel ones) at any nb, or the C operator sequence for an fp32 model or a pressure BC;
  * simulate.simulate: the operators called one by one from Python;
  * the oracle (oracle.simulate).
Before each step the operator copy and the oracle are re-seeded with the GPU's current state, so every comparison
covers exactly one step and the three see the same input.  Per step:
  (a) against the oracle: density bit for bit (advection and BCs are per-cell restatements); U and p within
      MODE_TOL of each batch entry's own max (the conv stack, test_gpu_step.py); the exact zeros of U are the
      oracle's;
  (b) against the operator sequence: density bit for bit; U and p within 1e-6 of each entry's max (the double
      atomics behind the input scale); the exact zeros of U and p are the same bits, sign included;
  (c) no trace fault.

The rows vary the shape (scalar kernels, every block width bx of the quad kernels, partial x and y blocks, odd nz),
the advection method and tile halo, the trace length, the optional state (density, velocity / density BCs, random
BCs with -0.0, unaligned views), the mconf (gravity, buoyancy, vorticity, strength, dt, a clamping input-scale
threshold), the flags (geometry, empty box, an open border, Empty / Outflow / Stick cells) and the conv mode.
test_case_table_reaches_every_branch (no GPU) keeps the table covering every branch of quad_dims
(tfl_fused.cu) and both paths of tfl_simulate_step, each at nb = 1 and nb > 1; test_case_paths_are_the_kernels_that_ran
proves each row's path from the kernels torch.profiler saw, so the restated rule cannot drift from the library's."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import oracle
from cases import bits_equal, describe_diff
from fluidnet_b200 import synth

MODE_TOL = {"fp32": 2e-5, "tf32x3": 2e-5, "tf32": 3e-3}
OPS_TOL = 1e-6
GRAVITY = [0.3, -0.8, 0.52]
BASE_MCONF = dict(dt=0.1, maccormackStrength=0.6, buoyancyScale=0.5, vorticityConfinementAmp=3.0,
                  simMethod="convnet")


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


CASES = {
    # the bench's path on a cube (quad kernels, bx = 8), plume BCs
    "cube32-plume": case((32, 32, 32)),
    # per-voxel kernels (nx / 4 = 5 quads): non-Ours methods, gravity, buoyancy
    "s12x14x20-euler": case((12, 14, 20), method="euler"),
    "s12x14x20-maccormack-gravity": case((12, 14, 20), method="maccormack", gravityScale=0.7, gravity=GRAVITY),
    "s12x14x20-rk3-random-tf32": case((12, 14, 20), method="rk3Ours", state="random", mode="tf32"),
    "s12x14x20-exotic": case((12, 14, 20), flags="exotic", amp=8.0),
    # bx = 4, partial y block, odd nz; density without BCs
    "q9x11x16-eulerOurs-density": case((9, 11, 16), method="eulerOurs", state="density"),
    # two x blocks (bx = 32), the second partial; velocity BC only; the two-kernel advection (tile mode 0)
    "q7x10x132-rk2Ours-ubc": case((7, 10, 132), method="rk2Ours", state="ubc"),
    "q7x10x132-tile0-amp8": case((7, 10, 132), tile=0, amp=8.0, gravityScale=0.4, gravity=GRAVITY),
    # bx = 2; random BCs (identity on some quads only, -0.0)
    "q16x12x8-rk3Ours-random": case((16, 12, 8), method="rk3Ours", state="random"),
    "q16x12x8-maccormack-random-tf32": case((16, 12, 8), method="maccormack", state="random", mode="tf32"),
    # bx = 1 (no left or right neighbour in a row), odd nz; no density and no BCs
    "q13x9x4-none": case((13, 9, 4), state="none", tile=0),
    # nz is the largest extent (getDx from z); tile halo 1, short traces; velocity BC without density
    "q40x12x16-tile1-amp2-ubc-nodens": case((40, 12, 16), tile=1, amp=2.0, state="ubc-nodens"),
    # bx = 16; tile halo 2 with traces of 0.8 cell and of 2.5 cells (beyond the halo)
    "q10x12x64-tile2-amp8": case((10, 12, 64), tile=2, amp=8.0, gravityScale=0.7, gravity=GRAVITY),
    "q10x12x64-tile2-amp25": case((10, 12, 64), tile=2, amp=25.0, state="random"),
    "q10x12x64-auto-amp25-euler": case((10, 12, 64), amp=25.0, method="euler", state="random"),
    # flags: Empty / Outflow / Stick cells, an empty box, an open border
    "q16x16x32-exotic": case((16, 16, 32), flags="exotic", state="random"),
    "q16x16x32-empty-box": case((16, 16, 32), flags="empty", gravityScale=1.0, gravity=GRAVITY),
    "q14x16x32-open-border": case((14, 16, 32), flags="open", tile=1, amp=2.0),
    # mconf: no vorticity, no buoyancy, full MacCormack strength, dt 0.25; an input scale clamped to the threshold
    "q12x16x32-novort-nobuoy-dt025": case((12, 16, 32), vorticityConfinementAmp=0.0, buoyancyScale=0.0,
                                          maccormackStrength=1.0, dt=0.25),
    "q12x16x32-threshold-tf32": case((12, 16, 32), threshold=50.0, mode="tf32"),
    # caller-owned views that are only 4-byte aligned: the per-voxel kernels on a quad shape
    "q12x16x32-unaligned": case((12, 16, 32), state="unaligned", method="eulerOurs"),
    # the fused step at nb = 2 with per-entry BCs (odd nz: no block straddles; test_gpu_batch_models.py has those)
    "q10x12x16-nb2": case((10, 12, 16), nb=2, method="maccormack"),
    # the C operator path: fp32 model, a pressure BC, each at nb = 1 and nb = 2
    "ops12x16x20-fp32": case((12, 16, 20), mode="fp32", gravityScale=0.5, gravity=GRAVITY),
    "ops16x16x16-pbc": case((16, 16, 16), pbc=True, method="rk2Ours"),
    "ops9x12x20-fp32-nb2": case((9, 12, 20), nb=2, mode="fp32", method="rk3Ours"),
    "ops8x12x16-pbc-nb2": case((8, 12, 16), nb=2, pbc=True, method="maccormack"),
}


# ---------------------------------------------------------------------------------------------------------------
# Which branch each case reaches (restated from tfl_simulate_step and quad_dims, tfl_fused.cu)
# ---------------------------------------------------------------------------------------------------------------
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


def branches(c):
    """The set of branch names this case reaches."""
    if not takes_fused_path(c):
        return {"ops"}
    nz, ny, nx = c["shape"]
    q = quad_dims(c["nb"], nz, ny, nx)
    if q is None or c["state"] == "unaligned":
        return {"fused", "scalar"}
    (gx, gy, _), (bx, by, bz) = q
    out = {"fused", "quad", "bx%d" % bx}
    if gx * bx * 4 > nx:
        out.add("partial-x")
    if gy * by > ny:
        out.add("partial-y")
    if bz == 2 and (c["nb"] * nz) % 2 == 1:
        out.add("odd-nz")
    return out


def test_case_table_reaches_every_branch():
    """No GPU: the table keeps reaching every block shape of the quad kernels, the per-voxel kernels and the C
    operator path, with every advection method and the optional state on the fused path."""
    reached = set()
    for c in CASES.values():
        reached |= branches(c)
    want = {"ops", "fused", "scalar", "quad", "partial-x", "partial-y", "odd-nz"} | {"bx%d" % b for b in
                                                                                     (1, 2, 4, 8, 16, 32)}
    assert want <= reached, sorted(want - reached)
    fused = [c for c in CASES.values() if takes_fused_path(c)]
    methods = {"euler", "maccormack", "eulerOurs", "rk2Ours", "rk3Ours", "maccormackOurs"}
    assert {c["method"] for c in fused if c["state"] not in ("none", "ubc-nodens")} == methods  # byte-flag scalar
    assert {c["tile"] for c in fused} == {None, 0, 1, 2}
    assert {c["amp"] for c in fused} >= {2.0, 8.0, 25.0}
    assert {c["state"] for c in fused} >= {"plume", "none", "density", "ubc", "ubc-nodens", "random", "unaligned"}
    assert {c["flags"] for c in fused} >= {"geom", "empty", "open", "exotic"}
    assert {c["mode"] for c in fused} == {"tf32x3", "tf32"}
    assert any(c["mconf"]["gravityScale"] > 0 for c in fused)
    assert any(c["mconf"]["vorticityConfinementAmp"] == 0 for c in fused)
    assert any(c["mconf"]["buoyancyScale"] == 0 for c in fused)
    assert any(c["threshold"] > 1.0 for c in fused)
    assert any(c["nb"] > 1 for c in fused)
    ops = [c for c in CASES.values() if not takes_fused_path(c)]
    for nb in (1, 2):                          # the operator path with each of its two reasons, alone and batched
        assert any(c["mode"] == "fp32" and c["nb"] == nb for c in ops), nb
        assert any(c["pbc"] and c["nb"] == nb for c in ops), nb
    # the scalar per-voxel kernels with buoyancy (k_post_advect's neighbour sums)
    assert any("scalar" in branches(c) and c["mconf"]["buoyancyScale"] > 0 and c["state"] != "none"
               for c in fused)


# ---------------------------------------------------------------------------------------------------------------
# State builders (numpy)
# ---------------------------------------------------------------------------------------------------------------
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


class LibraryOccupancyOracle(oracle.Oracle):
    """The oracle with the library's occupancy rule for flags that are neither exactly Fluid nor exactly Obstacle:
    -1 (k_cnn_inputs_fused*, k_cnn_inputs).  The CPU reference raises on such cells instead."""

    def flagsToOccupancy(self, flags):
        f = np.asarray(flags, np.float32)
        return np.where(f == synth.FLUID, 0.0, np.where(f == synth.OBSTACLE, 1.0, -1.0)).astype(np.float32)


# ---------------------------------------------------------------------------------------------------------------
# GPU helpers
# ---------------------------------------------------------------------------------------------------------------
def to_gpu(batch, unaligned=False):
    out = {}
    for k, v in batch.items():
        t = torch.from_numpy(v.copy()).cuda()
        if unaligned:
            flat = torch.empty(t.numel() + 1, device="cuda", dtype=t.dtype)
            view = flat[1:].view(t.shape)
            view.copy_(t)
            assert view.data_ptr() % 16 == 4 and view.is_contiguous()
            t = view
        out[k] = t
    return out


def set_tile_mode(mode):
    from fluidnet_b200 import tfluids
    ctx = tfluids.context()
    ctx.lib.tfl_debug_advect_tile.argtypes = [C.c_void_p, C.c_int]
    assert ctx.lib.tfl_debug_advect_tile(ctx.h, -1 if mode is None else mode) == 0


def host(batch):
    return {k: v.cpu().numpy() for k, v in batch.items()}


def close_per_entry(got, want, tol, what):
    for b in range(got.shape[0]):
        err = np.abs(got[b].astype(np.float64) - want[b].astype(np.float64)).max()
        scale = max(float(np.abs(want[b]).max()), 1e-6)
        assert err <= tol * scale, "%s[%d]: max err %g vs scale %g (tol %g)" % (what, b, err, scale, tol)


def same_zero_bits(got, want):
    z = (got == 0) | (want == 0)
    return np.array_equal(got[z].view(np.uint32), want[z].view(np.uint32))


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_step_paths(orc, name):
    from fluidnet_b200 import simulate, tfluids
    from gpu_backend import make_gpu_model
    c = CASES[name]
    batch = make_batch(orc, c)
    mnp = synth.make_model(True)
    gm = make_gpu_model(mnp, threshold=c["threshold"])
    gm.set_mode(c["mode"])
    mconf = c["mconf"]
    be = LibraryOccupancyOracle() if c["flags"] == "exotic" else orc
    unaligned = c["state"] == "unaligned"
    fused, ops = to_gpu(batch, unaligned), to_gpu(batch, unaligned)
    ctx = tfluids.context()
    set_tile_mode(c["tile"])
    try:
        ctx.trace_faults()
        be.lib.orc_reset_trace_faults()
        for step in range(3):
            ref = host(fused)
            for k in ops:
                ops[k].copy_(fused[k])
            oracle.simulate(be, mconf, ref, mnp)
            simulate.simulate_fused(None, mconf, fused, gm)
            simulate.simulate(None, mconf, ops, gm)
            got, opg = host(fused), host(ops)
            what = "%s step %d" % (name, step)
            if "density" in got:
                assert bits_equal(got["density"], ref["density"]), \
                    "%s density vs oracle: %s" % (what, describe_diff(got["density"], ref["density"]))
                assert bits_equal(got["density"], opg["density"]), \
                    "%s density vs ops: %s" % (what, describe_diff(got["density"], opg["density"]))
            for k in ("UDiv", "pDiv"):
                close_per_entry(got[k], ref[k], MODE_TOL[c["mode"]], "%s %s vs oracle" % (what, k))
                close_per_entry(got[k], opg[k], OPS_TOL, "%s %s vs ops" % (what, k))
                assert same_zero_bits(got[k], opg[k]), "%s %s: zeros differ from the operator sequence" % (what, k)
            assert np.array_equal(got["UDiv"] == 0, ref["UDiv"] == 0), "%s U: zeros differ from the oracle" % what
            assert ctx.trace_faults() == 0, what
        assert be.trace_faults() == 0, "the oracle traced out of the domain: the case is not a valid input"
    finally:
        set_tile_mode(None)


# ---------------------------------------------------------------------------------------------------------------
# Each row's path, from the kernels that ran
# ---------------------------------------------------------------------------------------------------------------
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


def expected_path(c):
    b = branches(c)
    return "ops" if "ops" in b else "scalar" if "scalar" in b else "quad"


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


def case_kernels():
    """{row: (launch tally, {kernel: count})} of one tfl_simulate_step per CASES row, under torch.profiler."""
    from fluidnet_b200 import simulate, tfluids
    from gpu_backend import make_gpu_model
    from test_gpu_launch_tally import _tally_and_kernels
    orc = oracle.Oracle()
    out = {}
    for name, c in CASES.items():
        gm = make_gpu_model(synth.make_model(True), threshold=c["threshold"])
        gm.set_mode(c["mode"])
        st = to_gpu(make_batch(orc, c), c["state"] == "unaligned")
        tally, kernels = _tally_and_kernels(tfluids.context(), lambda: simulate.simulate_fused(None, c["mconf"], st, gm),
                                            attempts=6)
        out[name] = (tally, dict(kernels))
    return out


@pytest.mark.gpu
def test_case_paths_are_the_kernels_that_ran():
    """Every row takes the path takes_fused_path and quad_dims restate (the fused step's quad or per-voxel kernels, or
    the operator sequence), as the profiler sees it; on the fused path the library's launch tally counts exactly those
    kernels."""
    seen = run_in_child("test_gpu_step_paths", "t.case_kernels()")
    assert set(seen) == set(CASES)
    for name, (tally, kernels) in seen.items():
        path = step_path(kernels)
        print("step path %s: %s (nb %d, %d kernels)" % (name, path, CASES[name]["nb"], tally))
        assert path == expected_path(CASES[name]), (name, path, sorted(kernels))
        if path != "ops":
            assert tally == sum(kernels.values()), (name, tally, kernels)


# ---------------------------------------------------------------------------------------------------------------
# The step graph: replays after in-place state changes, and refusal of a graph whose buffers were reallocated
# ---------------------------------------------------------------------------------------------------------------
def _scale_traces(b, cells):
    """U scaled so that its longest trace is `cells` cells (dt = 0.1)."""
    b["UDiv"].mul_(cells / 0.1 / b["UDiv"].abs().max())


GRAPH_EDITS = ("solid block on", "solid block off", "BC quads switched", "traces 2.5 cells", "pDiv")


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
        from gpu_backend import make_gpu_model
        self.use(ctx)
        m = make_gpu_model(mnp)
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


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(16, 12, 32), (12, 14, 20)], ids=["quad", "scalar"])
def test_step_graph_replays_follow_state_changes(orc, contexts, shape):
    """A graph captured once, then edited state between replays: flags (a solid block added, then removed: the
    replay must rebuild the clearance field), BC arrays (quads switched between identity and not: the replay must
    rebuild the quad mask), U (traces from 0.2 to 2.5 cells, past the tile halo chosen at capture) and pDiv.  Every
    replay equals, bit for bit, a direct step on a copy of the state driven through a second context, so that no
    flag cache, clearance or quad mask is shared: whatever the replay uses, it has built itself."""
    from fluidnet_b200 import simulate
    c = case(shape, state="random", amp=2.0)
    batch = make_batch(orc, c)
    mnp = synth.make_model(True)
    ctx_graph, ctx_ref = contexts.new(), contexts.new()
    gm_graph, gm_ref = contexts.model(ctx_graph, mnp), contexts.model(ctx_ref, mnp)
    mconf = c["mconf"]
    ref, gb = to_gpu(batch), to_gpu(batch)
    flags0 = ref["flags"].clone()
    nz, ny, nx = shape
    rs = np.random.RandomState(11)

    def edit(what, b):
        if what == "solid block on":
            b["flags"][..., nz // 4:nz // 2, ny // 2:ny - 2, 2:nx // 2] = synth.OBSTACLE
        elif what == "solid block off":
            b["flags"].copy_(flags0)
        elif what == "BC quads switched":
            nbc = {"UDiv": batch["UDiv"]}
            random_bcs(nbc, 77)
            for k in ("UBC", "UBCInvMask", "densityBC", "densityBCInvMask"):
                b[k].copy_(torch.from_numpy(nbc[k]))
        elif what == "traces 2.5 cells":
            _scale_traces(b, 2.5)
        else:
            b["pDiv"].copy_(torch.from_numpy(pdiv))

    def direct_step():
        contexts.use(ctx_ref)
        simulate.simulate_fused(None, mconf, ref, gm_ref)

    stream = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(stream):
        _scale_traces(ref, 0.2)
        _scale_traces(gb, 0.2)
        direct_step()
        contexts.use(ctx_graph)
        simulate.simulate_fused(None, mconf, gb, gm_graph)
        graph = simulate.StepGraph(mconf, gb, gm_graph)
        try:
            for what in ("",) + GRAPH_EDITS:
                pdiv = (rs.rand(*batch["pDiv"].shape).astype(np.float32) - np.float32(0.5)) * np.float32(0.2)
                if what:
                    edit(what, ref)
                    edit(what, gb)
                graph.launch()
                direct_step()
                stream.synchronize()
                for k in ("density", "UDiv", "pDiv"):
                    assert torch.equal(ref[k].view(torch.int32), gb[k].view(torch.int32)), (what, k)
        finally:
            graph.close()


@pytest.mark.gpu
def test_host_buffer_step_without_density(orc):
    """tfl_host_sim_step with density = NULL (no side stream, no density copies) returns what the device step
    without a density field leaves on the device."""
    from fluidnet_b200 import simulate, tfluids
    from gpu_backend import make_gpu_model
    c = case((32, 32, 32), state="ubc-nodens")
    batch = make_batch(orc, c)
    assert "density" not in batch
    gm = make_gpu_model(synth.make_model(True))
    mconf = c["mconf"]
    dev = to_gpu(batch)
    ctx = tfluids.context()
    lib = ctx.lib
    hs = C.c_void_p()
    keep = [np.ascontiguousarray(batch[k]) for k in ("flags", "UBC", "UBCInvMask")]
    nz, ny, nx = c["shape"]
    ctx.check(lib.tfl_host_sim_create(ctx.h, 1, nz, ny, nx, 1, *[a.ctypes.data for a in keep], None, None,
                                      C.byref(hs)))
    hp = torch.from_numpy(batch["pDiv"].copy()).pin_memory()
    hU = torch.from_numpy(batch["UDiv"].copy()).pin_memory()
    mc = simulate.make_mconf(mconf)
    mc.normalize_input_threshold = gm.threshold
    try:
        for step in range(3):
            simulate.simulate_fused(None, mconf, dev, gm)
            ctx.check(lib.tfl_host_sim_step(ctx.h, hs, hp.data_ptr(), hU.data_ptr(), None, C.byref(mc), gm.h))
            for k, h in (("UDiv", hU), ("pDiv", hp)):
                close_per_entry(h.numpy(), dev[k].cpu().numpy(), OPS_TOL, "step %d %s" % (step, k))
    finally:
        lib.tfl_host_sim_destroy(ctx.h, hs)


def _realloc_arena(gm):          # an operator on a larger grid grows the scratch arena
    from fluidnet_b200 import tfluids
    n = 64                       # advectVel needs 24 B per cell of scratch: 6.3 MB against the 32^3 step's 2.5 MB
    fl = torch.from_numpy(synth.make_flags(n, n, n, True)).cuda()
    U = torch.from_numpy(synth.make_smooth_velocity(fl.cpu().numpy(), True)).cuda()
    tfluids.advectVel(0.1, U, fl, "euler", torch.empty_like(U), 0.6)


def _realloc_flag_cache(gm):     # a traced advection on another (smaller) shape
    from fluidnet_b200 import tfluids
    fl = torch.from_numpy(synth.make_flags(20, 24, 16, True)).cuda()
    U = torch.from_numpy(synth.make_smooth_velocity(fl.cpu().numpy(), True)).cuda()
    tfluids.advectVel(0.1, U, fl, "maccormackOurs", torch.empty_like(U), 0.6)


def _realloc_activations(gm):    # the model on another grid
    n = 24
    fl = torch.from_numpy(synth.make_flags(n, n, n, True)).cuda()
    U = torch.from_numpy(synth.make_smooth_velocity(fl.cpu().numpy(), True)).cuda()
    gm.forward((torch.zeros_like(fl), U, fl))


@pytest.mark.gpu
@pytest.mark.parametrize("trigger,buffer", [(_realloc_arena, "scratch arena"), (_realloc_flag_cache, "flag cache"),
                                            (_realloc_activations, "activation buffers")],
                         ids=["arena", "flag-cache", "activations"])
def test_stale_step_graph_is_refused(orc, contexts, trigger, buffer):
    """A call that reallocates a buffer the graph captured makes tfl_step_graph_launch refuse the graph, naming the
    buffer, without replaying it; a graph captured again replays the direct step bit for bit."""
    from fluidnet_b200 import simulate
    from fluidnet_b200._lib import TflError
    c = case((32, 32, 32))
    batch = make_batch(orc, c)
    gm = contexts.model(contexts.new(), synth.make_model(True))     # a new context: its arena starts empty
    mconf = c["mconf"]
    ga, gb = to_gpu(batch), to_gpu(batch)
    stream = torch.cuda.Stream()
    torch.cuda.synchronize()

    def same():
        stream.synchronize()
        return all(torch.equal(ga[k].view(torch.int32), gb[k].view(torch.int32)) for k in ("density", "UDiv", "pDiv"))

    with torch.cuda.stream(stream):
        simulate.simulate_fused(None, mconf, ga, gm)
        simulate.simulate_fused(None, mconf, gb, gm)
        graph = simulate.StepGraph(mconf, gb, gm)
        graph.launch()
        simulate.simulate_fused(None, mconf, ga, gm)
        assert same()
        trigger(gm)
        with pytest.raises(TflError, match="stale graph: the (context|model)'s %s" % buffer):
            graph.launch()
        graph.close()
        assert same()                                  # the refused launch ran nothing
        simulate.simulate_fused(None, mconf, ga, gm)
        simulate.simulate_fused(None, mconf, gb, gm)   # re-sizes what the trigger changed
        graph = simulate.StepGraph(mconf, gb, gm)
        try:
            for _ in range(2):
                graph.launch()
                simulate.simulate_fused(None, mconf, ga, gm)
                assert same()
        finally:
            graph.close()
