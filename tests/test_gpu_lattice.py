"""Every advection dispatch of the library against the oracle, bit for bit, on the lattice inputs of
tests/lattice_cases.py: traces that end exactly on cell centres, faces, the domain ends and the faces of solids, and
trace lengths exactly at, and one or two ulps around, the thresholds of the trace loop (k + 1e-5), of the clear-space
fast paths (clearance - 0.51, clearance - 1.01) and of the tile halos (0.49, 1.49).  tests/test_oracle_lattice.py pins
the oracle on the reference's compiled CPU code at the same inputs.
  - the per-pass kernels (nb = 2, which the tile kernels do not take): all six methods, 2-D and 3-D, in place and out
    of place;
  - the 3-D maccormackOurs tile kernels, forced to the two-kernel version, halo 1, halo 2 and automatic, velocity and
    scalar with both sampleOutsideFluid settings; a forced halo must have launched its tile kernel;
  - the byte-flag instantiations inside tfl_simulate_step: the 'jacobi' step (bit for bit against the oracle's step),
    the fused convnet step (its density), and a replayed step graph of each;
  - emulated z-slabs at world 2 and 3 on 'jacobi', with z traces of exactly the margin's reach.
No call may count a trace fault."""
import ctypes as C

import numpy as np
import pytest
import torch

import lattice_cases as L
import oracle
from cases import bits_equal, describe_diff

pytestmark = pytest.mark.gpu

METHODS = list(oracle.ADVECT_METHODS)
CASES3 = [c for c in L.FIELD_CASES if c[1]]


@pytest.fixture(scope="module")
def gpu():
    from gpu_backend import GpuBackend
    return GpuBackend()


@pytest.fixture
def contexts():
    from step_cases import Contexts
    cs = Contexts()
    try:
        yield cs
    finally:
        cs.close()


def set_tile(ctx, mode):
    ctx.lib.tfl_debug_advect_tile.argtypes = [C.c_void_p, C.c_int]
    assert ctx.lib.tfl_debug_advect_tile(ctx.h, mode) == 0


def tile_used(ctx):
    f = ctx.lib.tfl_debug_advect_tile_used
    f.argtypes = [C.c_void_p, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_float)]
    v, s, t = C.c_int32(-1), C.c_int32(-1), C.c_float(-1.0)
    assert f(ctx.h, C.byref(v), C.byref(s), C.byref(t)) == 0
    return v.value, s.value, t.value


@pytest.mark.parametrize("case", L.FIELD_CASES, ids=L.FIELD_IDS)
def test_per_pass_kernels(orc, gpu, case):
    f = L.build(case, nb=2, wall_bcs=orc.setWallBcsForward)
    dt, U, fl, rho = f["dt"], f["U"], f["flags"], f["density"]
    gpu.trace_faults()
    for method in METHODS:
        want = orc.advectVel(dt, U, fl, method, 0.6)
        for in_place in (False, True):
            got = gpu.advectVel(dt, U, fl, method, 0.6, in_place=in_place)
            assert bits_equal(got, want), "advectVel %s in_place=%s: %s" % (method, in_place, describe_diff(got, want))
        for outside in (False, True):
            want = orc.advectScalar(dt, rho, U, fl, method, outside, 0.6)
            for in_place in (False, True):
                got = gpu.advectScalar(dt, rho, U, fl, method, outside, 0.6, in_place=in_place)
                assert bits_equal(got, want), "advectScalar %s outside=%s in_place=%s: %s" % (
                    method, outside, in_place, describe_diff(got, want))
    assert orc.trace_faults() == 0
    assert gpu.trace_faults() == 0


@pytest.mark.parametrize("case", CASES3, ids=[c[0] for c in CASES3])
def test_tile_kernels(orc, gpu, case):
    from fluidnet_b200 import tfluids
    ctx = tfluids.context()
    f = L.build(case, nb=1, wall_bcs=orc.setWallBcsForward)
    dt, U, fl, rho = f["dt"], f["U"], f["flags"], f["density"]
    census = L.tie_census(fl, U, dt)
    want_v = orc.advectVel(dt, U, fl, "maccormackOurs", 0.6)
    want_s = {o: orc.advectScalar(dt, rho, U, fl, "maccormackOurs", o, 0.6) for o in (False, True)}
    gpu.trace_faults()
    try:
        for mode in (0, 1, 2, -1):
            set_tile(ctx, mode)
            got = gpu.advectVel(dt, U, fl, "maccormackOurs", 0.6)
            assert bits_equal(got, want_v), "advectVel mode %d: %s (census %s)" % (mode, describe_diff(got, want_v),
                                                                                  census)
            vel_halo = tile_used(ctx)[0]
            for outside in (False, True):
                got = gpu.advectScalar(dt, rho, U, fl, "maccormackOurs", outside, 0.6)
                assert bits_equal(got, want_s[outside]), "advectScalar mode %d outside=%s: %s (census %s)" % (
                    mode, outside, describe_diff(got, want_s[outside]), census)
                if mode >= 0:
                    assert tile_used(ctx)[:2] == (mode, mode), (mode, vel_halo, tile_used(ctx))
            if mode >= 0:
                assert vel_halo == mode, (mode, vel_halo)
            got = gpu.advectVel(dt, U, fl, "maccormackOurs", 0.6, in_place=True)
            assert bits_equal(got, want_v), "advectVel in place, mode %d: %s" % (mode, describe_diff(got, want_v))
    finally:
        set_tile(ctx, -1)
    assert orc.trace_faults() == 0
    assert gpu.trace_faults() == 0


def step_batch(case, orc):
    f = L.build(case, nb=1, wall_bcs=orc.setWallBcsForward)
    return {"pDiv": np.zeros_like(f["flags"]), "UDiv": f["U"], "flags": f["flags"], "density": f["density"]}


def step_mconf(case, method):
    return oracle.default_mconf(dt=case[4], maccormackStrength=0.6, simMethod=method, maxIter=12, is3D=True,
                                vorticityConfinementAmp=0.5)


KEYS = ("pDiv", "UDiv", "density")
STEP_CASES = [c for c in CASES3 if c[2] in ("geom", "exotic")]
SLABS = [(2, 2), (2, 3), (3, 2)]        # (world, margin): three ranks of 20 planes are too thin for a margin of 3


@pytest.mark.parametrize("case", STEP_CASES, ids=[c[0] for c in STEP_CASES])
def test_step_and_graph(orc, contexts, case):
    """tfl_simulate_step and a replayed step graph on 'jacobi' (every field bit for bit against the oracle's step) and
    on the fused convnet step (density bit for bit).  The exotic flags run 'jacobi' only: the network's occupancy
    input is -1 on Empty / Outflow / Stick cells, where the oracle, like the CPU reference, raises."""
    from fluidnet_b200 import simulate, synth
    mnp = synth.make_model(True)
    for method in ("jacobi", "convnet") if case[2] != "exotic" else ("jacobi",):
        ctx = contexts.new()
        contexts.use(ctx)
        gm = contexts.model(ctx, mnp) if method == "convnet" else None
        batch = step_batch(case, orc)
        mconf = step_mconf(case, method)
        want = {k: v.copy() for k, v in batch.items()}
        oracle.simulate(orc, mconf, want, mnp if gm is not None else None)
        keys = KEYS if method == "jacobi" else ("density",)
        stream = torch.cuda.Stream()
        torch.cuda.synchronize()
        with torch.cuda.stream(stream):
            gb = {k: torch.from_numpy(v.copy()).cuda() for k, v in batch.items()}
            stream.synchronize()
            ctx.trace_faults()
            simulate.simulate_fused(None, mconf, gb, gm)
            stream.synchronize()
            for k in keys:
                got = gb[k].cpu().numpy()
                assert bits_equal(got, want[k]), "%s step, %s: %s" % (method, k, describe_diff(got, want[k]))
            graph = simulate.StepGraph(mconf, gb, gm)
            try:
                for k, v in batch.items():
                    gb[k].copy_(torch.from_numpy(v))
                graph.launch()
                stream.synchronize()
            finally:
                graph.close()
            for k in keys:
                got = gb[k].cpu().numpy()
                assert bits_equal(got, want[k]), "%s graph replay, %s: %s" % (method, k, describe_diff(got, want[k]))
        assert ctx.trace_faults() == 0, method
    assert orc.trace_faults() == 0


@pytest.mark.parametrize("world,margin", SLABS, ids=["world%d_margin%d" % s for s in SLABS])
def test_slabs_with_traces_of_the_margin(orc, contexts, world, margin):
    """z traces up to exactly margin - 1 cells (the reach a margin is documented for, ceil(max|u| dt) + 1) across
    rank boundaries: every emulated slab step equals the oracle's step bit for bit without a fault.  Traces of
    exactly margin cells: a step either counts a fault or equals it."""
    from fluidnet_b200.slab import SlabSimulator, run_lockstep
    flags = L.make_flags("geom", True)
    for reach, strict in ((margin - 1, True), (margin, False)):
        dt = 0.25
        U = L.make_velocity(flags, True, 2, dt, max_length=reach)
        orc.setWallBcsForward(U, flags)
        census = L.tie_census(flags, U, dt)
        assert float(np.abs(U).max()) * dt == reach and census["face"] > 0, census
        batch = {"pDiv": np.zeros_like(flags), "UDiv": U, "flags": flags, "density": L.density(flags)}
        mconf = oracle.default_mconf(dt=dt, maccormackStrength=0.6, simMethod="jacobi", maxIter=12, is3D=True)
        want = {k: v.copy() for k, v in batch.items()}
        oracle.simulate(orc, mconf, want, None)
        ctx = contexts.new()
        contexts.use(ctx)
        tb = {k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in batch.items()}
        sims = [SlabSimulator(tb, mconf, None, torch.device("cuda", 0), rank=r, world=world, margin=margin)
                for r in range(world)]
        ctx.trace_faults()
        run_lockstep(sims)
        faults = ctx.trace_faults()
        if strict or not faults:
            assert faults == 0, "world %d margin %d, traces up to %g: %d faults" % (world, margin, reach, faults)
            for k in KEYS:
                got = torch.cat([q.dec.owned(q.s[k]).cpu() for q in sims], dim=2).numpy()
                assert bits_equal(got, want[k]), "world %d margin %d, traces up to %g, %s: %s" % (
                    world, margin, reach, k, describe_diff(got, want[k]))
    assert orc.trace_faults() == 0
