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

import numpy as np
import pytest
import torch

import oracle
from cases import bits_equal, describe_diff
from fluidnet_b200 import synth
from step_cases import (MODE_TOL, OPS_TOL, case, close_per_entry, contexts, make_batch, quad_dims, random_bcs,
                        run_in_child, same_zero_bits, step_path, takes_fused_path)

GRAVITY = [0.3, -0.8, 0.52]


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


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_step_paths(orc, name):
    from fluidnet_b200 import simulate, tfluids
    from fluidnet_b200.model import ProjectionModel
    c = CASES[name]
    batch = make_batch(orc, c)
    mnp = synth.make_model(True)
    gm = ProjectionModel.from_model(mnp, normalizeInputThreshold=c["threshold"])
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


def expected_path(c):
    b = branches(c)
    return "ops" if "ops" in b else "scalar" if "scalar" in b else "quad"


def case_kernels():
    """{row: (launch tally, {kernel: count})} of one tfl_simulate_step per CASES row, under torch.profiler."""
    from fluidnet_b200 import simulate, tfluids
    from fluidnet_b200.model import ProjectionModel
    from step_cases import tally_and_kernels
    orc = oracle.Oracle()
    out = {}
    for name, c in CASES.items():
        gm = ProjectionModel.from_model(synth.make_model(True), normalizeInputThreshold=c["threshold"])
        gm.set_mode(c["mode"])
        st = to_gpu(make_batch(orc, c), c["state"] == "unaligned")
        tally, kernels = tally_and_kernels(tfluids.context(), lambda: simulate.simulate_fused(None, c["mconf"], st, gm),
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
    from fluidnet_b200.model import ProjectionModel
    c = case((32, 32, 32), state="ubc-nodens")
    batch = make_batch(orc, c)
    assert "density" not in batch
    gm = ProjectionModel.from_model(synth.make_model(True))
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
