"""The PCG step replayed from a step graph (tfl_step_graph_* with simMethod 'pcg'): the solve's iteration loop is a
conditional WHILE node the device re-arms, so the replay never returns to the host.

Every replay is held bit for bit (p, U and density as uint32) to tfl_simulate_step run from the same state, and every
tfl_step_graph_pcg_status to tfl_solve_linear_system_pcg on that step's divergence and flags:
  - pocket cases: 3-D components of every size class (1 cell: skipped, 2-4: no preconditioner, >= 5), 2-D with two
    batch entries, with and without density, with p / U boundary conditions;
  - the 64^3 plume of tests/long_run.py with simMethod 'pcg' (maxIter 34, as in the demo scene), 100 steps;
  - flags changed in place between replays: one component, then thousands of 2-cell pockets, then no fluid at all,
    then the start again;
  - the errors of the direct solve (a fluid cell on the border, a NaN in U), reported by pcg_status with the direct
    call's message, kept until read, gone after the next good replay;
  - two graphs on one context interleaved with direct solves, and the arena check after a larger direct solve;
  - tfl_launch_count against the direct step's and the device's iteration count."""
import numpy as np
import pytest
import torch

import long_run
import oracle
import pcg_cases
from cases import describe_diff
from fluidnet_b200 import simulate, synth, tfluids
from fluidnet_b200._lib import TflError

pytestmark = pytest.mark.gpu

KEYS = ("pDiv", "UDiv", "density")


@pytest.fixture
def contexts():
    from step_cases import Contexts
    cs = Contexts()
    try:
        cs.use(cs.new())
        yield cs
    finally:
        cs.close()


@pytest.fixture
def stream():
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        yield s
    s.synchronize()


def pcg_mconf(is3d, max_iter=34):
    return oracle.default_mconf(dt=0.1, maccormackStrength=0.6, buoyancyScale=1.0,
                                vorticityConfinementAmp=3.0 if is3d else 0.0, simMethod="pcg", maxIter=max_iter,
                                is3D=is3d)


def pocket_batch(orc, is3d, nb, density, bcs, seed=0):
    flags, U, _ = pcg_cases.make(orc, is3d, nb=nb, seed=seed)
    batch = {"pDiv": np.zeros_like(flags), "UDiv": U, "flags": flags}
    if density:
        batch["density"] = synth.make_density(flags)
    if bcs:
        inv = np.ones_like(flags)
        inv[..., 2:5, 2:6] = 0.0
        batch["pBCInvMask"] = inv
        batch["pBC"] = np.where(inv == 0, np.float32(0.05), np.float32(0.0)).astype(np.float32)
        uinv = np.ones_like(U)
        uinv[..., 10:12, 3:5] = 0.0
        batch["UBCInvMask"] = uinv
        batch["UBC"] = np.where(uinv == 0, np.float32(0.25), np.float32(0.0)).astype(np.float32)
    return {k: np.ascontiguousarray(v, np.float32) for k, v in batch.items()}


def to_gpu(batch):
    return {k: torch.from_numpy(v.copy()).cuda() for k, v in batch.items()}


def same(ga, gb, what):
    for k in KEYS:
        if k in ga:
            a, b = ga[k], gb[k]
            assert torch.equal(a.view(torch.int32), b.view(torch.int32)), "%s, %s: %s" % (
                what, k, describe_diff(a.cpu().numpy(), b.cpu().numpy()))


def capture(mconf, batch):
    """(ga, gb, graph): two copies of the state, each stepped once directly; graph = the step captured on gb."""
    ga, gb = to_gpu(batch), to_gpu(batch)
    simulate.simulate_fused(None, mconf, ga)
    simulate.simulate_fused(None, mconf, gb)
    return ga, gb, simulate.StepGraph(mconf, gb)


def direct_status(gb, mconf, is3d):
    """(residual, iterations, p) of tfl_solve_linear_system_pcg on the divergence and flags the last step left."""
    p = torch.empty_like(gb["pDiv"])
    res = tfluids.solveLinearSystemPCG(p, gb["flags"], gb["div"], is3d, 1e-4, mconf["maxIter"], "ic0")
    return res, tfluids.solveLinearSystemPCG.last_iterations, p


def step_both(ga, graph, mconf):
    simulate.simulate_fused(None, mconf, ga)
    graph.launch()


POCKETS = [("3d-pockets-density", True, 1, True, False), ("3d-pockets-nodensity", True, 1, False, False),
           ("3d-pockets-bcs", True, 1, True, True), ("2d-nb2-density", False, 2, True, False),
           ("2d-nb2-bcs", False, 2, False, True)]


@pytest.mark.parametrize("case", POCKETS, ids=[c[0] for c in POCKETS])
def test_replay_equals_the_step(orc, contexts, stream, case):
    _, is3d, nb, density, bcs = case
    mconf = pcg_mconf(is3d)
    ga, gb, graph = capture(mconf, pocket_batch(orc, is3d, nb, density, bcs))
    try:
        for i in range(3):
            step_both(ga, graph, mconf)
            stream.synchronize()
            same(ga, gb, "replay %d" % (i + 1))
            res, it = graph.pcg_status()
            want_res, want_it, _ = direct_status(gb, mconf, is3d)
            assert (res, it) == (want_res, want_it) and it > 0
    finally:
        graph.close()


def test_long_plume_run(contexts, stream):
    """100 replays against 100 direct steps, bit for bit after every step; pcg_status against the direct solve of the
    step's own divergence, whose p must also be the step's (the plume has no pressure BC)."""
    mconf = long_run.make_mconf(True, "pcg")
    mconf["maxIter"] = 34
    batch = long_run.make_batch(True)
    ga, gb = to_gpu(batch), to_gpu(batch)
    simulate.simulate_fused(None, mconf, ga)      # step 1 direct on both, then the graph from step 2
    simulate.simulate_fused(None, mconf, gb)
    graph = simulate.StepGraph(mconf, gb)
    its = []
    try:
        for step in range(2, long_run.N + 1):
            step_both(ga, graph, mconf)
            res, it = graph.pcg_status()
            same(ga, gb, "step %d" % step)
            want_res, want_it, p = direct_status(gb, mconf, True)
            assert (res, it) == (want_res, want_it), (step, res, it, want_res, want_it)
            assert torch.equal(p.view(torch.int32), gb["pDiv"].view(torch.int32)), step
            its.append(it)
    finally:
        graph.close()
    assert 0 < min(its) and max(its) <= 35           # iter <= maxIter: at most maxIter + 1


def pockets_of_two(n):
    """[1][1][n][n][n] flags: obstacles everywhere but pairs of fluid cells along x on odd (z, y) rows."""
    f = np.full((1, 1, n, n, n), 2.0, np.float32)
    for x0 in range(1, n - 2, 4):
        f[0, 0, 1:n - 1:2, 1:n - 1:2, x0:x0 + 2] = 1.0
    return f


def test_flags_changed_in_place(orc, contexts, stream):
    n = 48
    mconf = pcg_mconf(True)
    start = synth.make_flags(n, n, n, True, nb=1, geometry=False)
    U = synth.make_smooth_velocity(start, True, amp=2.0)
    orc.setWallBcsForward(U, start)
    batch = {"pDiv": np.zeros_like(start), "UDiv": U, "flags": start, "density": synth.make_density(start)}
    pockets = pockets_of_two(n)
    assert (pockets == 1).sum() // 2 > 5000
    ga, gb, graph = capture(mconf, batch)
    try:
        for what, flags in (("one component", start), ("pockets", pockets),
                            ("no fluid", np.full_like(start, 2.0)), ("start again", start)):
            t = torch.from_numpy(flags).cuda()
            ga["flags"].copy_(t)
            gb["flags"].copy_(t)
            for i in range(2):
                step_both(ga, graph, mconf)
                stream.synchronize()
                same(ga, gb, "%s, replay %d" % (what, i + 1))
                res, it = graph.pcg_status()
                want = direct_status(gb, mconf, True)
                assert (res, it) == want[:2], (what, res, it, want[:2])
                if what == "no fluid":
                    assert (res, it) == (float("-inf"), 0)
                    assert not gb["pDiv"].any()
                elif what == "one component":
                    assert it > 0
    finally:
        graph.close()


@pytest.mark.parametrize("fault", ["border", "nan"])
def test_errors_are_reported_and_sticky(orc, contexts, stream, fault):
    mconf = pcg_mconf(True)
    batch = pocket_batch(orc, True, 1, True, True)
    f = batch["flags"][0, 0]
    inner = (f == 1)
    for axis in range(3):
        for shift in (1, -1):
            inner &= np.roll(f, shift, axis) == 1
    cell = tuple(int(v[0]) for v in np.nonzero(inner))          # a fluid cell with six fluid neighbours
    ga, gb, graph = capture(mconf, batch)
    try:
        good = {k: gb[k].clone() for k in gb}

        def spoil(b):
            if fault == "border":
                b["flags"][0, 0, 0, 5, 5] = 1.0
            else:              # a velocity BC writes it into U after the advection (whose clamp would drop it)
                b["UBCInvMask"][(0, 1) + cell] = 0.0
                b["UBC"][(0, 1) + cell] = float("nan")

        def restore(b):
            for k in good:
                b[k].copy_(good[k])

        spoil(ga)
        with pytest.raises(TflError) as direct:
            simulate.simulate_fused(None, mconf, ga)
        msg = str(direct.value)
        assert ("border" in msg) if fault == "border" else ("nan" in msg)
        spoil(gb)
        for _ in range(2):
            graph.launch()                 # the replay itself cannot fail
        restore(gb)
        restore(ga)
        step_both(ga, graph, mconf)         # a good replay does not clear the unread error
        stream.synchronize()
        same(ga, gb, "good replay after the error")
        with pytest.raises(TflError) as replayed:
            graph.pcg_status()
        assert str(replayed.value) == msg
        step_both(ga, graph, mconf)
        res, it = graph.pcg_status()        # read once: gone
        same(ga, gb, "second good replay")
        assert (res, it) == direct_status(gb, mconf, True)[:2]
    finally:
        graph.close()


def test_two_graphs_and_direct_solves(orc, contexts, stream):
    mconf = pcg_mconf(True)
    ga, gb, graph_b = capture(mconf, pocket_batch(orc, True, 1, True, False, seed=0))
    ha, hb, graph_h = capture(mconf, pocket_batch(orc, True, 1, True, False, seed=1))
    flags, _, div = pcg_cases.make(orc, True, nb=1, seed=2)
    fl, dv = torch.from_numpy(flags).cuda(), torch.from_numpy(div).cuda()
    want_p = np.zeros_like(flags)
    try:
        for i in range(3):
            step_both(ga, graph_b, mconf)
            p = torch.zeros_like(fl)
            tfluids.solveLinearSystemPCG(p, fl, dv, True, 1e-4, 34, "ic0")
            if i == 0:
                want_p = p.cpu().numpy()
            step_both(ha, graph_h, mconf)
            stream.synchronize()
            same(ga, gb, "graph 1, replay %d" % (i + 1))
            same(ha, hb, "graph 2, replay %d" % (i + 1))
            assert np.array_equal(p.cpu().numpy().view(np.uint32), want_p.view(np.uint32))
            assert graph_b.pcg_status() == direct_status(gb, mconf, True)[:2]
            assert graph_h.pcg_status() == direct_status(hb, mconf, True)[:2]
        big_flags, _, big_div = pcg_cases.make(orc, True, nb=2, seed=3, n=(40, 36, 30))
        tfluids.solveLinearSystemPCG(torch.zeros_like(torch.from_numpy(big_flags)).cuda(),
                                     torch.from_numpy(big_flags).cuda(), torch.from_numpy(big_div).cuda(), True,
                                     1e-4, 34, "ic0")
        for g in (graph_b, graph_h):
            with pytest.raises(TflError, match="arena"):
                g.launch()
    finally:
        graph_b.close()
        graph_h.close()


def test_refusals_and_other_methods(orc, contexts, stream):
    mconf = pcg_mconf(True)
    batch = pocket_batch(orc, True, 1, True, False)
    flags = np.ones((1, 1, 4, 970, 6), np.float32)
    oracle.Oracle().emptyDomain(flags, True, 1)
    wide = {"pDiv": np.zeros_like(flags), "UDiv": np.zeros((1, 3, 4, 970, 6), np.float32), "flags": flags}
    with pytest.raises(TflError, match="ny > 960"):
        simulate.StepGraph(mconf, to_gpu(wide))
    jm = dict(mconf, simMethod="jacobi")
    gb = to_gpu(batch)
    simulate.simulate_fused(None, jm, gb)
    graph = simulate.StepGraph(jm, gb)
    try:
        graph.launch()
        assert graph.pcg_status()[1] == -1
    finally:
        graph.close()


def test_launch_tally(orc, contexts, stream):
    """tfl_launch_count stays exact.  torch.profiler does not report the kernels of a conditional body reliably (on
    driver 580 it showed one pass of the body per replay, and memset / memcpy nodes as kernels named memset32 /
    memcpy32_post), so a replay is checked against the direct step from the same state: it must count what the direct
    step runs minus the iterations of pcg_solve's host loop (four per read-back, 4 kernels each: sweep, direction,
    update, scalars) plus the captured driver's own three kernels outside the loop (k_comp_clear, the first
    k_pcg_continue, k_pcg_finish).  pcg_status then adds ceil(iterations / 2) passes of 2 x 4 + 1 kernels (two
    iterations and the loop test), iterations being the longest component's count the device reports."""
    mconf = pcg_mconf(True)
    ga, gb, graph = capture(mconf, pocket_batch(orc, True, 1, True, False))
    ctx = tfluids._ctx_for(gb["pDiv"])
    try:
        for _ in range(3):
            c0 = ctx.launch_count()
            simulate.simulate_fused(None, mconf, ga)
            direct = ctx.launch_count() - c0
            c1 = ctx.launch_count()
            graph.launch()
            stream.synchronize()
            outside = ctx.launch_count() - c1
            c2 = ctx.launch_count()
            _, it = graph.pcg_status()
            assert it > 2
            assert outside == direct - 16 * ((it + 3) // 4) + 3, (outside, direct, it)
            assert ctx.launch_count() - c2 == (it + 1) // 2 * 9
            same(ga, gb, "tally replay")
    finally:
        graph.close()
