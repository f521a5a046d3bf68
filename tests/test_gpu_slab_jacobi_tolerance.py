"""simMethod 'jacobi' on z-slabs solved to a tolerance (tfl_slab_sim_set_jacobi_tolerance): the step must equal the
whole-grid operator sequence with solveLinearSystemJacobiDevice as its solve -- owned p, U and density bit for bit, the
same iteration count, the residual within 1e-6 relative -- at one rank in one process and with one process per rank on
cuda:0 (the harness of test_gpu_slab_ranks.py), where the residual's bits must also be the same at every world size.
Stops on the first sweep, inside a block (the block runs again from its start), on a block's last sweep (the 1-plane
p exchange), on the last sweep allowed and never.  Every pTol lies more than 1e-5 relative away from every residual the
solve tests, so the two residuals' summation orders cannot decide differently."""
import contextlib
import ctypes as C
import math
import time

import pytest
import torch
import torch.multiprocessing as mp

from slab_cases import KEYS, Comm, TIMEOUT_S, collect, jacobi_problem

pytestmark = pytest.mark.gpu

GAP = 1e-5
HALO = 6                                    # margin 2


def _residuals(solve, flags, div, is3d, max_iter):
    """The whole-grid solve's residual after each sweep (the host loop with pTol = 0 reports its last sweep's)."""
    p = torch.empty_like(div)
    return [solve(p, flags, div, is3d, 0, k) for k in range(1, max_iter + 1)]


def _stop_sweep(res, p_tol, max_iter):
    """(0-based sweep the loop stops after, iteration count)."""
    for s, r in enumerate(res):
        if r < p_tol:
            return s, s
        if s + 1 >= max_iter:
            return s, s + 1
    raise AssertionError("no stop")


def _tol_for(res, target):
    """A pTol that stops the loop after sweep `target` (None: never), GAP away from every residual before it."""
    if target is None:
        return min(res) * 0.5
    hi = min(res[:target]) if target > 0 else res[0] * 4
    lo = res[target]
    assert lo < hi * (1 - 4 * GAP), "residuals do not fall at sweep %d: %r" % (target, res[:target + 1])
    return math.sqrt(lo * hi)


@contextlib.contextmanager
def _whole_grid_dev_solve(p_tol, log):
    """simulate.simulate with solveLinearSystemJacobiDevice(pTol) as its Jacobi solve; `log` receives per call the
    (residual, iterations, residual of every sweep up to the stop)."""
    from fluidnet_b200 import tfluids
    orig = tfluids.solveLinearSystemJacobi

    def solve(p, flags, div, is3D, pTol=None, maxIter=None, verbose=None):
        res_all = _residuals(orig, flags, div, is3D, maxIter)
        r, it = tfluids.solveLinearSystemJacobiDevice(p, flags, div, is3D, p_tol, maxIter)
        log.append((float(r.item()), int(it.item()), res_all))
        return float(r.item())

    tfluids.solveLinearSystemJacobi = solve
    try:
        yield
    finally:
        tfluids.solveLinearSystemJacobi = orig


def _reference(tb, mconf, p_tol, steps):
    from fluidnet_b200 import simulate
    gb = {k: v.cuda() for k, v in tb.items()}
    out, log = [], []
    with _whole_grid_dev_solve(p_tol, log):
        for _ in range(steps):
            simulate.simulate(None, mconf, gb)
            out.append({k: gb[k].cpu().clone() for k in KEYS})
    return out, log


def _gap_ok(res_all, p_tol, stop):
    return all(abs(r - p_tol) > GAP * p_tol for r in res_all[:stop + 1])


def _first_step_residuals(tb, mconf):
    _, log = _reference(tb, mconf, 1e-30, 1)
    return log[0][2]


# (nx, ny, gnz, maxIter, target stop sweep: int, "last" = maxIter - 1, None = never)
TARGETS = [0, 2, 5, 13, "last", None]
SHAPES = [(128, 16, 24), (32, 24, 20)]


@pytest.mark.parametrize("target", TARGETS, ids=lambda t: "stop%s" % t)
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "nx%d" % s[0])
def test_world1_equals_whole_grid_dev_solve(shape, target):
    from fluidnet_b200.slab import NativeSlabSimulator
    nx, ny, gnz = shape
    max_iter = 20
    tb, mconf = jacobi_problem(nx, ny, gnz, max_iter=max_iter)
    res0 = _first_step_residuals(tb, mconf)
    p_tol = _tol_for(res0, max_iter - 1 if target == "last" else target)
    want, log = _reference(tb, mconf, p_tol, 3)
    assert _stop_sweep(res0, p_tol, max_iter)[0] == (max_iter - 1 if target in ("last", None) else target)
    sim = NativeSlabSimulator(tb, mconf, None, torch.device("cuda", 0), rank=0, world=1)
    sim.set_jacobi_tolerance(p_tol)
    for step in range(3):
        sim.step()
        res, it = sim.jacobi_status()
        w_res, w_it, res_all = log[step]
        if not _gap_ok(res_all, p_tol, _stop_sweep(res_all, p_tol, max_iter)[0]):
            assert step > 0, "pTol %g too close to a first-step residual" % p_tol
            break
        assert it == w_it, (step, it, w_it)
        assert abs(res - w_res) <= 1e-6 * abs(w_res), (step, res, w_res)
        for k in KEYS:
            assert torch.equal(sim.gather(k), want[step][k]), "step %d %s" % (step, k)
        assert sim.jacobi_stats()[0] == 0
    sim.check()
    sim.close()


def _plume_sim(tb, mconf, p_tol):
    from fluidnet_b200.slab import NativeSlabSimulator
    sim = NativeSlabSimulator(tb, mconf, None, torch.device("cuda", 0), rank=0, world=1)
    sim.set_jacobi_tolerance(p_tol)
    return sim


def test_world1_graph_replays_equal_direct_steps():
    """Replays interleaved with direct steps equal an all-direct run bit for bit over 12 plume steps whose iteration
    counts differ; the replay's host time stays at the fixed-count replay's; a replay counts its loop body once."""
    from fluidnet_b200.slab import SlabStepGraph
    tb, mconf = jacobi_problem(128, 16, 24, max_iter=24)
    res0 = _first_step_residuals(tb, mconf)
    p_tol = _tol_for(res0, 8)
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        direct, mixed = _plume_sim(tb, mconf, p_tol), _plume_sim(tb, mconf, p_tol)
        direct.step()
        mixed.step()
        l0 = mixed.ctx.launch_count()
        graph = SlabStepGraph(mixed)
        assert mixed.ctx.launch_count() == l0
        iters, deltas = [], []
        for step in range(12):
            direct.step()
            l0 = mixed.ctx.launch_count()
            if step % 3 != 1:
                graph.launch()
                deltas.append(mixed.ctx.launch_count() - l0)
            else:
                mixed.step()
            a, b = direct.jacobi_status(), mixed.jacobi_status()
            assert a == b, (step, a, b)
            iters.append(a[1])
            for k in KEYS:
                assert torch.equal(direct.gather(k), mixed.gather(k)), "step %d %s" % (step, k)
        assert len(set(iters)) > 1, iters
        assert len(set(deltas)) == 1, deltas
        # the graph is block 0, one pass of the WHILE body and the last block: a direct step that enqueues three
        # blocks (chunks of 1 and 2) launches as many kernels
        sims = {}
        for target in (8, 15):
            if _stop_sweep(res0, _tol_for(res0, target), 24)[0] // HALO not in (1, 2):
                continue
            s = _plume_sim(tb, mconf, _tol_for(res0, target))
            l0 = s.ctx.launch_count()
            s.step()
            sims[target] = s.ctx.launch_count() - l0
            s.close()
        assert sims and all(v == deltas[0] for v in sims.values()), (sims, deltas)
        # host time around a replay: the fixed-count replay of the same step is the yardstick
        fixed = _plume_sim(tb, mconf, p_tol)
        fixed.set_jacobi_tolerance(0.0)
        fixed.step()
        fgraph = SlabStepGraph(fixed)

        def host_ms(g):
            ts = []
            for _ in range(9):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                g.launch()
                ts.append((time.perf_counter() - t0) * 1e3)
            torch.cuda.synchronize()
            return sorted(ts)[4]

        host_ms(graph), host_ms(fgraph)
        t_tol, t_fixed = host_ms(graph), host_ms(fgraph)
        assert t_tol <= 3 * t_fixed + 0.2, (t_tol, t_fixed)
        for g in (graph, fgraph):
            g.close()
        for s in (direct, mixed, fixed):
            s.close()


def test_zero_tolerance_after_a_tolerance_is_the_fixed_step():
    tb, mconf = jacobi_problem(32, 24, 20, max_iter=20)
    res0 = _first_step_residuals(tb, mconf)
    a = _plume_sim(tb, mconf, _tol_for(res0, 7))
    a.step()
    a.set_jacobi_tolerance(0.0)
    b = _plume_sim(tb, mconf, 0.0)
    st = a.download()
    b.ctx.check(b.ctx.lib.tfl_slab_sim_upload(b.ctx.h, b.h, st["pDiv"].ctypes.data, st["UDiv"].ctypes.data,
                                              st["density"].ctypes.data))
    counts = []
    for s in (a, b):
        l0 = s.ctx.launch_count()
        s.step()
        counts.append(s.ctx.launch_count() - l0)
    assert counts[0] == counts[1], counts
    for k in KEYS:
        assert torch.equal(a.gather(k), b.gather(k)), k
    assert a.jacobi_stats()[1] >= 0.0
    a.close()
    b.close()


def test_refusals_name_their_cause_and_launch_nothing():
    from fluidnet_b200._lib import TflError
    tb, mconf = jacobi_problem(32, 24, 16, max_iter=5)
    sim = _plume_sim(tb, mconf, 0.0)
    lib, h = sim.ctx.lib, sim.ctx.h

    def refused(call, words):
        l0 = sim.ctx.launch_count()
        with pytest.raises(TflError, match=words):
            call()
        assert sim.ctx.launch_count() == l0, "a refused call launched work"

    for bad in (-1e-3, float("nan")):
        refused(lambda: sim.set_jacobi_tolerance(bad), "pTol must be >= 0")
    refused(sim.jacobi_status, "no step has solved to a Jacobi tolerance")
    sim.step()                                          # a fixed-count step does not count
    refused(sim.jacobi_status, "no step has solved to a Jacobi tolerance")
    sim.set_jacobi_tolerance(1e-4)
    sim.step()
    sim.jacobi_status()
    sim.set_jacobi_tolerance(0.0)                       # the status of an earlier tolerance step is not this step's
    sim.step()
    refused(sim.jacobi_status, "ran the fixed count")
    sim.set_jacobi_tolerance(1e-4)
    sim.step()
    sim.jacobi_status()
    g = torch.cuda.CUDAGraph()
    x = torch.zeros(4, device="cuda")
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        sim.ctx.use_current_stream()                    # the context's stream is the one captured below
    l0 = sim.ctx.launch_count()
    with torch.cuda.graph(g, stream=side, capture_error_mode="relaxed"):
        x.add_(1)
        res, it = C.c_float(), C.c_int32()
        rc = lib.tfl_slab_sim_jacobi_status(h, sim.h, C.byref(res), C.byref(it))
        msg = lib.tfl_last_error(h)
        rc_step = lib.tfl_slab_sim_step(h, sim.h, C.byref(sim.mc), None)
        msg_step = lib.tfl_last_error(h)
    assert rc != 0 and b"captured" in msg, msg
    assert rc_step != 0 and b"tfl_slab_graph_create" in msg_step, msg_step
    assert sim.ctx.launch_count() == l0
    sim.close()


# ---- one process per rank on cuda:0 --------------------------------------------------------------------------------
def _want_p_traffic(gnz, ny, nx, world, rank, max_iter, stop):
    """(p exchanges, bytes) of a solve that stops after global sweep `stop`."""
    from fluidnet_b200.slab import jacobi_schedule
    _, blocks = jacobi_schedule(gnz, world, rank, 2, max_iter)
    b, s = stop // HALO, stop % HALO
    widths = [blocks[i][1] for i in range(1, b + 1)]
    # a stop on the last sweep of a block leaves p stale below the owned planes, except in the schedule's last block
    fix = s == blocks[b][0] - 1 and b < len(blocks) - 1
    planes = sum(widths) + (1 if fix else 0)
    nbrs = (rank > 0) + (rank < world - 1)
    return len(widths) + (1 if fix else 0), planes * ny * nx * 4 * nbrs


def _cases(world):
    # (nx, ny, gnz, maxIter, stop targets over the steps' first-step residuals, skew, graph)
    return [(128, 16, 6 * world + 1, 20, 2, False, False),
            (32, 24, 6 * world + 5, 20, 5, True, False),
            (128, 16, 6 * world + 3, 20, 13, False, True),
            (32, 24, 6 * world + 1, 14, None, False, False),
            # maxIter a multiple of the halo: the schedule closes with the 1-plane exchange alone, which a stop at
            # maxIter on the last block's last sweep reproduces
            (128, 16, 6 * world + 2, 18, None, False, True)]


def _rank_worker(rank, world, q, qd, inboxes, barrier):
    try:
        from fluidnet_b200.slab import NativeSlabSimulator, SlabStepGraph
        torch.cuda.set_device(0)
        comm = Comm(rank, world, inboxes)
        wait = lambda: barrier.wait(TIMEOUT_S)       # noqa: E731
        fails = []
        for ci, (nx, ny, gnz, max_iter, target, skew, use_graph) in enumerate(_cases(world)):
            tb, mconf = jacobi_problem(nx, ny, gnz, max_iter=max_iter)
            if rank == 0:
                res0 = _first_step_residuals(tb, mconf)
                p_tol = _tol_for(res0, target)
                want, log = _reference(tb, mconf, p_tol, 3)
                one = _plume_sim(tb, mconf, p_tol)          # world 1: the residual bits every world must give
                one_status = []
                for _ in range(3):
                    one.step()
                    one_status.append(one.jacobi_status())
                one.close()
            p_tol = comm.allgather(p_tol if rank == 0 else None)[0]
            stream = torch.cuda.Stream()
            with torch.cuda.stream(stream):
                sim = NativeSlabSimulator(tb, mconf, None, torch.device("cuda", 0), rank, world, margin=2,
                                          allgather=comm.allgather, barrier=wait)
                sim.set_jacobi_tolerance(p_tol)
                graph = None
                got = []
                for step in range(3):
                    if skew and rank == step % world:
                        time.sleep(0.03)
                    if graph is not None and (step + rank) % 2 == 0:
                        graph.launch()
                    else:
                        sim.step()
                    if use_graph and graph is None:
                        graph = SlabStepGraph(sim)
                    status = sim.jacobi_status()
                    n, ms, by = sim.jacobi_stats()
                    d = sim.download()
                    got.append((status, n, by, {k: d[k][:, :, sim.z0:sim.z1].copy() for k in KEYS}))
                torch.cuda.synchronize()
                faults = sim.ctx.trace_faults()
                if graph is not None:
                    graph.close()
                sim.close()
            if faults:
                fails.append("case %d rank %d: %d faults" % (ci, rank, faults))
            for step, (status, n, by, _) in enumerate(got):
                stop = status[1] if status[0] < p_tol else status[1] - 1
                want_n, want_by = _want_p_traffic(gnz, ny, nx, world, rank, max_iter, stop)
                if (n, by) != (want_n, want_by):
                    fails.append("case %d rank %d step %d: p exchanges %r, the stop says %r" % (
                        ci, rank, step, (n, by), (want_n, want_by)))
            qd.put((ci, rank, sim.z0, sim.z1, [(g[0], g[3]) for g in got]))
            if rank == 0:
                parts = {}
                while len(parts) < world:
                    c, r, z0, z1, per_step = qd.get(timeout=TIMEOUT_S)
                    parts[r] = (z0, z1, per_step)
                for step in range(3):
                    w_res, w_it, res_all = log[step]
                    if not _gap_ok(res_all, p_tol, _stop_sweep(res_all, p_tol, max_iter)[0]):
                        if step == 0:
                            fails.append("case %d: pTol %g too close to a first-step residual" % (ci, p_tol))
                        break
                    for r, (z0, z1, per_step) in parts.items():
                        (res, it), arrs = per_step[step]
                        if (res, it) != one_status[step] or it != w_it or abs(res - w_res) > 1e-6 * abs(w_res):
                            fails.append("case %d step %d rank %d: status %r, world 1 %r, whole grid %r" % (
                                ci, step, r, (res, it), one_status[step], (w_res, w_it)))
                        for k in KEYS:
                            if not torch.equal(torch.from_numpy(arrs[k]), want[step][k][:, :, z0:z1]):
                                fails.append("case %d step %d rank %d: %s differs" % (ci, step, r, k))
            wait()
        q.put((rank, "ok", fails))
    except Exception:               # pragma: no cover
        import traceback
        q.put((rank, "FAIL: %s" % traceback.format_exc(), []))
        raise


@pytest.mark.parametrize("world", [2, 3, 4])
def test_ranks_equal_whole_grid_dev_solve(world):
    ctx = mp.get_context("spawn")
    q, qd, barrier = ctx.Queue(), ctx.Queue(), ctx.Barrier(world)
    inboxes = [ctx.Queue() for _ in range(world)]
    procs = [ctx.Process(target=_rank_worker, args=(r, world, q, qd, inboxes, barrier)) for r in range(world)]
    for p in procs:
        p.start()
    res = collect(procs, q, TIMEOUT_S)
    assert len(res) == world and all(r[1] == "ok" for r in res), res
    fails = [f for r in res for f in r[2]]
    assert not fails, "\n".join(fails)
