"""The step over the long plume run of tests/long_run.py (N = 100 steps at 64^3, and at 128^2), against the oracle.

The Jacobi path is a per-cell restatement of the oracle, so every run below is held to the oracle's trajectory bit for
bit after every step, through every regime of the advection-tile halo choice (halo 1, halo 2, the two-kernel version
and its probes of the halo-2 kernel):
  (a) tfl_simulate_step with the automatic tile halo, whose choices tfl_debug_advect_tile_used reports;
  (b) the same with the halo forced to each mode (two-kernel, 1, 2);
  (c) the per-operator step, simulate.simulate;
  (d) a step graph captured after step 1 (halo 1) and replayed to N, recording every third density frame into a
      three-slot FrameRecorder behind the replays;
  (e) step graphs captured at the first step of the halo-2 and of the two-kernel regime, replayed from there to N;
  2-D: (a), (c) and (d) on the 128^2 run (no tile kernels; the 2-D quad and Jacobi kernels).
The convnet path (3xTF32 projection network) diverges chaotically from the oracle at the 1e-6 level, so it is held to
one step from the GPU's own state at steps 1, N/2 and N, and its graph replay to the direct step bit for bit.
z-slabs (two and three emulated ranks on one GPU) follow the trajectory bit for bit with a margin sized from its
velocities, and with a margin the velocities outgrow they are never silently wrong: a step either counts a fault or
equals the single-GPU step.

The oracle's 3-D trajectory takes about 8 s on the host (0.065 s per 64^3 step on 8 cores), the 2-D one under a second;
the whole module ran in 22 s on one H100 (80 GB HBM3, 700 W power limit)."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import long_run
import oracle
from cases import bits_equal, describe_diff
from fluidnet_b200 import synth

pytestmark = pytest.mark.gpu

N = long_run.N
KEYS = long_run.KEYS


@pytest.fixture(scope="module")
def traj3d():
    return long_run.oracle_trajectory(oracle.Oracle(), True)


@pytest.fixture(scope="module")
def traj2d():
    return long_run.oracle_trajectory(oracle.Oracle(), False)


@pytest.fixture
def contexts():
    from test_gpu_step_paths import Contexts
    cs = Contexts()
    try:
        yield cs
    finally:
        cs.close()


def fresh(contexts):
    """A library context of its own (tile telemetry at zero, no probe count) that tfluids calls through."""
    ctx = contexts.new()
    contexts.use(ctx)
    return ctx


def to_gpu(batch, state):
    b = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in batch.items() if k not in KEYS}
    b.update({k: torch.from_numpy(state[k].copy()).cuda() for k in KEYS})
    return b


def expect(gb, want, step, what):
    for k in KEYS:
        got = gb[k].cpu().numpy()
        assert bits_equal(got, want[k]), "%s: first difference after step %d, %s: %s" % (
            what, step, k, describe_diff(got, want[k]))


def set_tile_mode(ctx, mode):
    ctx.lib.tfl_debug_advect_tile.argtypes = [C.c_void_p, C.c_int, C.c_int]
    assert ctx.lib.tfl_debug_advect_tile(ctx.h, mode, 0) == 0


def tile_used(ctx):
    """(halo of the last advectVel tile launch, of the last advectScalar one, longest trace in the telemetry)."""
    f = ctx.lib.tfl_debug_advect_tile_used
    f.argtypes = [C.c_void_p, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_float)]
    v, s, t = C.c_int32(-1), C.c_int32(-1), C.c_float(-1.0)
    assert f(ctx.h, C.byref(v), C.byref(s), C.byref(t)) == 0
    return v.value, s.value, t.value


def run_direct(traj, ctx, what, is3d=True, fused=True, on_step=None):
    from fluidnet_b200 import simulate
    batch, states = traj
    mconf = long_run.make_mconf(is3d)
    gb = to_gpu(batch, states[0])
    ctx.trace_faults()
    for s in range(1, N + 1):
        (simulate.simulate_fused if fused else simulate.simulate)(None, mconf, gb, None)
        torch.cuda.synchronize()
        if on_step:
            on_step(s)
        expect(gb, states[s], s, what)
    assert ctx.trace_faults() == 0, what


# ---------------------------------------------------------------------------------------------------------------
# Jacobi path, bit for bit at every step
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def auto_halos(traj3d):
    """Run (a): the automatic tile halo on a fresh context.  Returns {step: (velocity halo, scalar halo, longest
    trace reported after the step)}."""
    from test_gpu_step_paths import Contexts
    cs = Contexts()
    try:
        ctx = fresh(cs)
        used = {}
        run_direct(traj3d, ctx, "tfl_simulate_step, automatic tile halo",
                   on_step=lambda s: used.__setitem__(s, tile_used(ctx)))
        return used
    finally:
        cs.close()


def test_jacobi_automatic_halo_visits_every_regime(auto_halos):
    used = auto_halos
    vel = {s: used[s][0] for s in used}
    assert vel[1] == 1 and used[1][1] == 1, "the first step must run the halo-1 tile kernels: %s" % (used[1],)
    assert set(vel.values()) == {0, 1, 2}, "velocity halos used: %s" % sorted(set(vel.values()))
    first2 = min(s for s in vel if vel[s] == 2)
    first0 = min(s for s in vel if vel[s] == 0)
    assert first2 < first0, (first2, first0)
    # a probe: the halo-2 kernel after a step that reported a trace beyond 1.4 cells
    probes = [s for s in range(2, N + 1) if vel[s] == 2 and used[s - 1][2] >= 1.4]
    assert probes, "no probe of the halo-2 kernel in %d two-kernel calls" % sum(v == 0 for v in vel.values())
    assert probes[0] == first0 + 15, "two-kernel regime from step %d, probes at steps %s" % (first0, probes)
    # the density runs on the halo chosen from the previous step's velocity trace, and never probes
    assert {used[s][1] for s in used} == {0, 1, 2}
    assert all(used[s][1] == 0 for s in probes)


@pytest.mark.parametrize("mode", [0, 1, 2], ids=["two-kernel", "halo1", "halo2"])
def test_jacobi_forced_tile_mode(traj3d, contexts, mode):
    ctx = fresh(contexts)
    set_tile_mode(ctx, mode)
    run_direct(traj3d, ctx, "tfl_simulate_step, tile mode %d" % mode)


def test_jacobi_operator_sequence(traj3d, contexts):
    ctx = fresh(contexts)
    run_direct(traj3d, ctx, "simulate.simulate", fused=False)


def replay(traj, ctx, start, what, is3d=True, expect_halo=None, record=False):
    """Direct steps from states[start] to start + 1, a step graph captured there and replayed to N.  record: every
    third density frame through a three-slot FrameRecorder, each taken frame against the oracle's density."""
    from fluidnet_b200 import record as frec, simulate
    batch, states = traj
    mconf = long_run.make_mconf(is3d)
    stream = torch.cuda.Stream()
    torch.cuda.synchronize()
    frames = []
    with torch.cuda.stream(stream):
        gb = to_gpu(batch, states[start])
        stream.synchronize()
        ctx.trace_faults()
        simulate.simulate_fused(None, mconf, gb, None)
        expect(gb, states[start + 1], start + 1, what + " (direct step)")
        graph = simulate.StepGraph(mconf, gb, None)
        if expect_halo is not None:
            assert tile_used(ctx)[0] == expect_halo, (what, tile_used(ctx))
        rec = frec.FrameRecorder(gb["density"].shape, slots=3) if record else None
        pending = []

        def take():
            idx, frame = rec.take(wait=True)
            s = pending.pop(0)
            want = states[s]["density"][0, 0].transpose(2, 1, 0)
            assert np.array_equal(frame.view(np.uint32), want.view(np.uint32)), \
                "%s: recorded frame %d (step %d) differs from the oracle's density" % (what, idx, s)
            rec.release()
            frames.append(s)

        try:
            for s in range(start + 2, N + 1):
                graph.launch()
                if rec is not None and s % 3 == 0:
                    if rec.full:
                        take()
                    rec.capture(gb["density"])
                    pending.append(s)
                expect(gb, states[s], s, what)
            while rec is not None and pending:
                take()
        finally:
            graph.close()
            if rec is not None:
                rec.close()
        stream.synchronize()
    assert ctx.trace_faults() == 0, what
    return frames


def test_jacobi_graph_from_step_1_with_recorder(traj3d, contexts):
    ctx = fresh(contexts)
    frames = replay(traj3d, ctx, 0, "step graph captured after step 1", expect_halo=1, record=True)
    assert frames == list(range(3, N + 1, 3))          # the ring of 3 wrapped len(frames) / 3 times


@pytest.mark.parametrize("halo", [2, 0], ids=["halo2", "two-kernel"])
def test_jacobi_graph_captured_in_later_regime(traj3d, auto_halos, contexts, halo):
    """Captured at the first step run (a) took with this halo: a direct step first, so that the telemetry the
    capture reads is that of the step before, as in (a)."""
    first = min(s for s in auto_halos if auto_halos[s][0] == halo)
    ctx = fresh(contexts)
    replay(traj3d, ctx, first - 2, "step graph captured at step %d (halo %d)" % (first, halo), expect_halo=halo)


def test_jacobi_2d(traj2d, contexts):
    ctx = fresh(contexts)

    def no_tile_kernel(s):
        assert tile_used(ctx)[:2] == (0, 0), "step %d ran a tile kernel on a 2-D grid" % s

    run_direct(traj2d, ctx, "2-D tfl_simulate_step", is3d=False, on_step=no_tile_kernel)
    run_direct(traj2d, fresh(contexts), "2-D simulate.simulate", is3d=False, fused=False)
    replay(traj2d, fresh(contexts), 0, "2-D step graph captured after step 1", is3d=False)


# ---------------------------------------------------------------------------------------------------------------
# Convnet path: graph replay bit for bit, one step from the GPU's own state at steps 1, N/2 and N
# ---------------------------------------------------------------------------------------------------------------
def close(got, want, tol, what):
    err = np.abs(got.astype(np.float64) - want.astype(np.float64)).max()
    scale = max(float(np.abs(want).max()), 1e-6)
    assert err <= tol * scale, "%s: max err %g vs scale %g (tol %g)" % (what, err, scale, tol)


def test_convnet_long_run(orc, contexts):
    from fluidnet_b200 import simulate
    ctx = fresh(contexts)
    mnp = synth.make_model(True)
    gm = contexts.model(ctx, mnp)
    assert gm.get_mode() == "tf32x3"
    batch = long_run.make_batch(True)
    mconf = long_run.make_mconf(True, "convnet")
    checkpoints = (1, N // 2, N)
    host = lambda b: {k: b[k].cpu().numpy() for k in KEYS}
    stream = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(stream):
        direct = to_gpu(batch, batch)
        graphed = to_gpu(batch, batch)
        stream.synchronize()
        ctx.trace_faults()
        before = {}
        graph = None
        try:
            for s in range(1, N + 1):
                if s in checkpoints:
                    before[s] = host(direct)
                simulate.simulate_fused(None, mconf, direct, gm)
                if graph is None:
                    simulate.simulate_fused(None, mconf, graphed, gm)
                    graph = simulate.StepGraph(mconf, graphed, gm)
                else:
                    graph.launch()
                stream.synchronize()
                for k in KEYS:
                    assert torch.equal(direct[k].view(torch.int32), graphed[k].view(torch.int32)), \
                        "graph replay differs from tfl_simulate_step after step %d, %s" % (s, k)
        finally:
            if graph is not None:
                graph.close()
        assert ctx.trace_faults() == 0
        for s in checkpoints:
            # the fused step from the state before step s, against the oracle and the operator sequence
            fused = to_gpu(batch, before[s])
            ops = to_gpu(batch, before[s])
            simulate.simulate_fused(None, mconf, fused, gm)
            simulate.simulate(None, mconf, ops, gm)
            got, opg = host(fused), host(ops)
            ref = {k: v.copy() for k, v in batch.items() if k not in KEYS}
            ref.update({k: before[s][k].copy() for k in KEYS})
            oracle.simulate(orc, mconf, ref, mnp)
            what = "convnet step %d" % s
            assert bits_equal(got["density"], ref["density"]), \
                "%s density vs oracle: %s" % (what, describe_diff(got["density"], ref["density"]))
            for k in ("UDiv", "pDiv"):
                close(got[k], ref[k], 2e-5, "%s %s vs oracle" % (what, k))
                close(got[k], opg[k], 1e-6, "%s %s vs the operator sequence" % (what, k))
            assert bits_equal(got["density"], opg["density"]), what
        stream.synchronize()
    assert ctx.trace_faults() == 0
    # the plume has accelerated: the late checkpoints step a state faster than the first
    assert long_run.trace_proxy(before[N]["UDiv"]) > 2 * long_run.trace_proxy(before[1]["UDiv"])


# ---------------------------------------------------------------------------------------------------------------
# z-slabs (emulated ranks on one GPU)
# ---------------------------------------------------------------------------------------------------------------
def slab_sims(traj, world, margin):
    from fluidnet_b200.slab import SlabSimulator
    batch, states = traj
    tb = {k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in batch.items() if k not in KEYS}
    tb.update({k: torch.from_numpy(states[0][k].copy()) for k in KEYS})
    return [SlabSimulator(tb, long_run.make_mconf(True), None, torch.device("cuda", 0), rank=r, world=world,
                          margin=margin) for r in range(world)]


def gathered(sims, k):
    return torch.cat([q.dec.owned(q.s[k]).cpu() for q in sims], dim=2).numpy()


@pytest.mark.parametrize("world", [2, 3])
def test_slabs_with_margin_from_the_velocities(traj3d, contexts, world):
    """margin = ceil(max |u| dt) + 1 over the whole run: every step equals the single-GPU trajectory (= the oracle's,
    which the tests above hold it to), and the fault counter that SlabSimulator.check reads stays at zero."""
    from fluidnet_b200.slab import run_lockstep
    batch, states = traj3d
    margin = math.ceil(max(long_run.trace_proxy(s["UDiv"]) for s in states)) + 1
    assert margin > 2
    ctx = fresh(contexts)
    sims = slab_sims(traj3d, world, margin)
    assert all(q.ctx is ctx for q in sims)
    ctx.trace_faults()
    for s in range(1, N + 1):
        run_lockstep(sims)
        for k in KEYS:
            got = gathered(sims, k)
            assert bits_equal(got, states[s][k]), "world %d margin %d: first difference after step %d, %s: %s" % (
                world, margin, s, k, describe_diff(got, states[s][k]))
        assert ctx.trace_faults() == 0, "world %d margin %d: fault counted at step %d" % (world, margin, s)


@pytest.mark.parametrize("world", [2, 3])
def test_slabs_outgrown_margin_is_never_silent(traj3d, contexts, world):
    """The default margin (2): at every step either a fault is counted (SlabSimulator.check would raise) or the
    gathered fields equal the single-GPU step from the same state.  The run's own z-traces stay within about a cell,
    so after the N steps the velocity is scaled up until the margin is outgrown, with a single-GPU step on its own
    context alongside; a fault must be counted there."""
    from fluidnet_b200 import simulate
    from fluidnet_b200.slab import run_lockstep
    batch, states = traj3d
    mconf = long_run.make_mconf(True)
    ref_ctx = contexts.new()
    ctx = fresh(contexts)
    sims = slab_sims(traj3d, world, 2)
    ctx.trace_faults()
    faulted = None

    def step_and_check(s, want):
        run_lockstep(sims)
        faults = ctx.trace_faults()
        if faults:
            return True
        for k in KEYS:
            got = gathered(sims, k)
            assert bits_equal(got, want[k]), \
                "world %d margin 2, step %s: %s differs from the single-GPU step and no fault was counted: %s" % (
                    world, s, k, describe_diff(got, want[k]))
        return False

    for s in range(1, N + 1):
        if step_and_check(s, states[s]):
            faulted = s
            break
    scale = 1.0
    while faulted is None and scale < 8:
        # continue from the (bit-identical) state with every velocity scaled: longer z-traces every step
        scale *= 1.5
        ref = to_gpu(batch, {k: gathered(sims, k) for k in KEYS})
        for q in sims:
            q.s["UDiv"].mul_(1.5)
        ref["UDiv"].mul_(1.5)
        contexts.use(ref_ctx)
        simulate.simulate(None, mconf, ref, None)
        contexts.use(ctx)
        torch.cuda.synchronize()
        if step_and_check("N + scale %.2f" % scale, {k: ref[k].cpu().numpy() for k in KEYS}):
            faulted = scale
    assert faulted is not None, "the default margin was never outgrown"
