"""The step monitor (tfl_monitor_*, monitor.py): its values against the oracle's divergence and a host restatement of
its reduction order, records after direct steps and replayed step graphs, records that never make the host wait, its
refusals, z-slab records combined over ranks (processes sharing cuda:0), and the scene's --stats file."""
import os
import time

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

import monitor_reference as ref
import oracle
from fluidnet_b200 import monitor, scene, simulate, synth, tfluids
from fluidnet_b200._lib import TflError
from fluidnet_b200.model import ProjectionModel
from scenes import plume_batch, step_mconf

pytestmark = pytest.mark.gpu

TIMEOUT_S = 400


def _fields(is3d, nb, shape, seed):
    nz, ny, nx = shape
    flags = synth.make_flags(nx, ny, nz, is3d, nb=nb, geometry=True, exotic=True, seed=seed)
    U = synth.make_velocity(flags, is3d, amp=3.0, seed=seed + 1)
    return U, flags


@pytest.mark.parametrize("is3d,nb,shape", [(True, 2, (30, 36, 40)), (False, 2, (1, 80, 72)), (True, 1, (7, 3, 5))])
def test_values_match_the_oracle_and_the_plane_ordered_restatement(is3d, nb, shape):
    U, flags = _fields(is3d, nb, shape, seed=11)
    orc = oracle.Oracle()
    div = orc.velocityDivergenceForward(U, flags)
    batch = {"UDiv": torch.from_numpy(U).cuda(), "flags": torch.from_numpy(flags).cuda()}
    with monitor.StepMonitor(None, batch, capacity=4) as mon:
        assert mon.record(batch) == 0 and mon.record(batch) == 1
        (i0, a), (i1, b) = mon.take(), mon.take()
    assert (i0, i1) == (0, 1)
    assert a.tobytes() == b.tobytes(), "the same fields gave different bits"
    for e in range(nb):
        assert a[e, 1] == float(np.abs(div[e]).max())
        assert a[e, 2] == float(np.abs(U[e]).max())
        want = np.sqrt(np.sum(div[e].astype(np.float64) ** 2))
        assert abs(a[e, 0] - want) <= 1e-12 * want
    assert a.tobytes() == ref.totals(ref.plane_partials(div, U)).tobytes()


def test_nan_propagates_into_every_maximum():
    """A field that went NaN shows in div_max and u_max, not only in div_norm; a NaN in a non-fluid cell (d = 0 there)
    only in u_max."""
    U, flags = _fields(True, 1, (12, 10, 9), seed=13)
    interior = U.copy()
    interior[0, 1, 6, 5, 4] = np.nan                     # a fluid cell of the synthetic grid: d is NaN there
    assert flags[0, 0, 6, 5, 4] == 1
    border = U.copy()
    border[0, 0, 0, 3, 3] = np.nan                       # the bottom plane is an obstacle border: d = 0
    got = []
    for u in (interior, border):
        batch = {"UDiv": torch.from_numpy(u).cuda(), "flags": torch.from_numpy(flags).cuda()}
        with monitor.StepMonitor(None, batch, capacity=1) as mon:
            mon.record(batch)
            got.append(mon.take()[1][0])
    assert np.isnan(got[0]).all(), got[0]
    assert np.isfinite(got[1][:2]).all() and np.isnan(got[1][2]), got[1]
    p = np.zeros((1, 4, 3))
    p[0, 2, 1] = np.nan
    from fluidnet_b200.monitor import combine_planes
    assert np.isnan(combine_planes([(0, p[:, :2]), (2, p[:, 2:])])[0, 1])


def _plume(n, sim_method):
    return plume_batch(n, inflow=n / 128.0), step_mconf(n, simMethod=sim_method, maxIter=34)


def _run_path(batch_np, mconf, model, steps, graph):
    """Records after every step (direct fused steps, or one fused step and then graph replays) and the fields
    downloaded after each."""
    stream = torch.cuda.Stream()
    recs, fields = [], []
    with torch.cuda.stream(stream):
        gb = {k: torch.from_numpy(v.copy()).cuda() for k, v in batch_np.items()}
        g = None
        with monitor.StepMonitor(None, gb, capacity=steps) as mon:
            for i in range(steps):
                if g is not None:
                    g.launch()
                else:
                    simulate.simulate_fused(None, mconf, gb, model)
                mon.record(gb)
                fields.append((gb["UDiv"].cpu().numpy(), gb["flags"].cpu().numpy()))
                if graph and i == 0:
                    g = simulate.StepGraph(mconf, gb, model)
            recs = mon.drain(wait=True)
        if g is not None:
            g.close()
    return [r[1] for r in recs], fields


@pytest.mark.parametrize("sim_method", ["convnet", "jacobi", "pcg"])
def test_records_of_direct_steps_and_step_graph_replays(sim_method):
    batch, mconf = _plume(64, sim_method)
    model = ProjectionModel(synth.make_model(True)["layers"], True) if sim_method == "convnet" else None
    orc = oracle.Oracle()
    direct, fd = _run_path(batch, mconf, model, 30, graph=False)
    replay, fr = _run_path(batch, mconf, model, 30, graph=True)
    for step in range(30):
        for recs, fields, what in ((direct, fd, "direct"), (replay, fr, "replayed")):
            want = ref.record(orc, *fields[step])
            assert recs[step].tobytes() == want.tobytes(), "%s step %d: %r, the fields give %r" % (
                what, step, recs[step], want)
        assert all(np.array_equal(a, b) for a, b in zip(fd[step], fr[step])), \
            "step %d: the replay's fields differ from the direct step's" % step
        assert direct[step].tobytes() == replay[step].tobytes(), step


def test_record_and_take_do_not_wait_for_the_device():
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        U, flags = _fields(True, 1, (64, 64, 64), seed=3)
        batch = {"UDiv": torch.from_numpy(U).cuda(), "flags": torch.from_numpy(flags).cuda()}
        mon = monitor.StepMonitor(None, batch, capacity=2)
        a = torch.randn(4096, 4096, device="cuda")
        b = torch.randn(4096, 4096, device="cuda") / 64.0
        with monitor.StepMonitor(None, batch, capacity=1) as warm:     # the kernels and the matmul loaded beforehand
            warm.record(batch)
            warm.take(wait=True)
        a = a @ b
        stream.synchronize()
        for _ in range(20):                            # ~50 ms of ordinary matmuls queued ahead of the record
            a = a @ b
        t0 = time.perf_counter()
        assert mon.record(batch) == 0
        returned = time.perf_counter() - t0
        assert not stream.query(), "the queued work finished before the record returned: nothing was measured"
        t0 = time.perf_counter()
        assert mon.take(wait=False) is None
        took = time.perf_counter() - t0
        assert not stream.query()
        stream.synchronize()
        got = mon.take(wait=False)
        assert got is not None and got[0] == 0
        assert got[1].tobytes() == ref.record(oracle.Oracle(), U, flags).tobytes()
        mon.close()
    assert returned < 0.02, returned
    assert took < 0.02, took


def test_refusals_name_their_cause_and_launch_nothing():
    ctx = tfluids.context()
    U, flags = _fields(True, 1, (8, 8, 8), seed=5)
    batch = {"UDiv": torch.from_numpy(U).cuda(), "flags": torch.from_numpy(flags).cuda()}
    with monitor.StepMonitor(None, batch, capacity=1) as mon:
        l0 = ctx.launch_count()
        with pytest.raises(TflError, match="holds no record"):
            mon.take(wait=True)
        two = {k: v.repeat(2, 1, 1, 1, 1) for k, v in batch.items()}
        with pytest.raises(TflError, match="nb = 2"):
            mon.record(two)
        deeper = {k: torch.cat([v, v], dim=2) for k, v in batch.items()}
        with pytest.raises(TflError, match="gnz = 16"):
            mon.record(deeper)
        with pytest.raises(TflError, match="shape mismatch"):
            mon.record({"UDiv": batch["UDiv"][:, :, :, :, :4].contiguous(), "flags": batch["flags"]})
        s = torch.cuda.Stream()
        g = torch.cuda.CUDAGraph()
        x = torch.zeros(4, device="cuda")
        with torch.cuda.stream(s):
            x.add_(1)
            ctx.use_current_stream()            # adopting a stream synchronises the old one: not inside the capture
            s.synchronize()
            with torch.cuda.graph(g, stream=s):
                x.add_(1)
                with pytest.raises(TflError, match="being captured"):
                    mon.record(batch)
        assert ctx.launch_count() == l0
        mon.record(batch)
        wider = {k: torch.cat([v, v], dim=4) for k, v in batch.items()}
        with pytest.raises(TflError, match="slot"):
            mon.record(batch)
        mon.take()
        with pytest.raises(TflError, match="differs from the monitor's first record"):
            mon.record(wider)
        assert ctx.launch_count() == l0 + 2


# ---- z-slabs -------------------------------------------------------------------------------------------------------
SLAB_STEPS = 40
FRAME_STEPS = 12


def _slab_problem(kind):
    from slab_cases import jacobi_problem
    tb, mconf = jacobi_problem(48, 48, 48, max_iter=34)
    if kind == "convnet":
        mconf = dict(mconf, simMethod="convnet")
    return tb, mconf


def _slab_worker(rank, world, kinds, q, qd, inboxes, barrier):
    try:
        from slab_cases import Comm
        from fluidnet_b200.slab import NativeSlabSimulator
        torch.cuda.set_device(0)
        comm = Comm(rank, world, inboxes)
        wait = lambda: barrier.wait(TIMEOUT_S)       # noqa: E731
        faults = 0
        for kind in kinds:
            tb, mconf = _slab_problem(kind)
            layers = synth.make_model(True)["layers"] if kind == "convnet" else None
            sim = NativeSlabSimulator(tb, mconf, layers, torch.device("cuda", 0), rank, world, margin=3,
                                      conv_mode="tf32x3" if layers else None, allgather=comm.allgather, barrier=wait)
            mon = sim.monitor(capacity=4)
            for step in range(SLAB_STEPS):
                sim.step()
                mon.record()
                idx, rec = mon.take()
                U = sim.download()["UDiv"][:, :, sim.z0:sim.z1].copy() if kind == "convnet" else None
                qd.put((kind, step, rank, idx, rec, sim.z0, sim.z1, U))
            torch.cuda.synchronize()
            faults += sim.ctx.trace_faults()
            mon.close()
            if kind == "jacobi":
                faults += _frames_without_waits(sim, rank, world, qd)
            sim.close()
        q.put((rank, "ok", faults))
    except Exception:               # pragma: no cover
        import traceback
        q.put((rank, "FAIL: %s" % traceback.format_exc(), 0))
        raise


def _frames_without_waits(sim, rank, world, qd):
    """The scene's per-frame path over several ranks, continuing the run: record_frame after every step with a ring of
    4 records, each step followed by ~25 ms of queued matmuls.  A record_frame that synchronised the stream (as an
    object gather through torch.distributed does) would leave it drained; taking a full ring's oldest record may wait
    for that record, never for the work behind it.  collect() at the end gathers once."""
    mon = sim.monitor(capacity=4)
    a = torch.randn(4096, 4096, device="cuda")
    b = torch.randn(4096, 4096, device="cuda") / 64.0
    slow = []
    stream = torch.cuda.current_stream()
    for step in range(FRAME_STEPS):
        sim.step()
        for _ in range(10):
            a = a @ b
        mon.record_frame()
        if stream.query():
            slow.append(step)
    recs = mon.collect()
    torch.cuda.synchronize()
    faults = sim.ctx.trace_faults()
    mon.close()
    qd.put(("frames", 0, rank, [r[0] for r in recs], [r[1] for r in recs], slow, None, None))
    return faults


def _whole_grid_records(tb, mconf, steps):
    """The whole-grid monitor after every step of the single-GPU operator sequence."""
    gb = {k: v.cuda() for k, v in tb.items()}
    out = []
    with monitor.StepMonitor(None, gb, capacity=steps) as mon:
        for _ in range(steps):
            simulate.simulate(None, mconf, gb)
            mon.record(gb)
        out = [r[1] for r in mon.drain(wait=True)]
    return out


def test_slab_records_equal_the_whole_grid_monitor_at_one_rank():
    from fluidnet_b200.slab import NativeSlabSimulator
    tb, mconf = _slab_problem("jacobi")
    want = _whole_grid_records(tb, mconf, SLAB_STEPS)
    sim = NativeSlabSimulator(tb, mconf, None, torch.device("cuda", 0), 0, 1, margin=3)
    with sim.monitor(capacity=3) as mon:
        got = []
        for _ in range(SLAB_STEPS):
            sim.step()
            if mon.full:
                got.append(mon.take())
            mon.record()
        got += mon.drain()
    sim.check()
    sim.close()
    assert [i for i, _ in got] == list(range(SLAB_STEPS))
    for step, (_, rec) in enumerate(got):
        assert rec.tobytes() == want[step].tobytes(), (step, rec, want[step])


@pytest.mark.parametrize("world", [2, 3])
def test_slab_records_over_processes_sharing_one_gpu(world):
    """'jacobi': the combined records equal the single-GPU whole-grid monitor bit for bit, every step.  'convnet' (world
    2): they equal the monitor of that run's gathered fields."""
    from slab_cases import collect
    kinds = ["jacobi", "convnet"] if world == 2 else ["jacobi"]
    tb, mconf = _slab_problem("jacobi")
    allw = _whole_grid_records(tb, mconf, SLAB_STEPS + FRAME_STEPS)
    want, want_more = allw[:SLAB_STEPS], allw[SLAB_STEPS:]
    torch.cuda.synchronize()
    ctx = mp.get_context("spawn")
    q, qd, barrier = ctx.Queue(), ctx.Queue(), ctx.Barrier(world)
    inboxes = [ctx.Queue() for _ in range(world)]
    procs = [ctx.Process(target=_slab_worker, args=(r, world, kinds, q, qd, inboxes, barrier)) for r in range(world)]
    for p in procs:
        p.start()
    got = {}
    while len(got) < (len(kinds) * SLAB_STEPS + 1) * world:
        kind, step, rank, idx, rec, z0, z1, U = qd.get(timeout=TIMEOUT_S)
        got[(kind, step, rank)] = (idx, rec, z0, z1, U)
    res = collect(procs, q, TIMEOUT_S)
    assert len(res) == world and all(r[1] == "ok" for r in res), res
    assert sum(r[2] for r in res) == 0, "trace faults: %r" % res
    orc = oracle.Oracle()
    flags = tb["flags"].numpy()
    for kind in kinds:
        for step in range(SLAB_STEPS):
            parts = [got[(kind, step, r)] for r in range(world)]
            assert all(p[0] == step for p in parts)
            assert all(p[1].tobytes() == parts[0][1].tobytes() for p in parts), "ranks disagree at step %d" % step
            if kind == "jacobi":
                w = want[step]
            else:
                U = np.concatenate([p[4] for p in sorted(parts, key=lambda p: p[2])], axis=2)
                w = ref.record(orc, np.ascontiguousarray(U), flags)
            assert parts[0][1].tobytes() == w.tobytes(), (kind, step, parts[0][1], w)
    for r in range(world):                   # the per-frame path: no waits, one gather, the whole grid's records
        idx, recs, slow = got[("frames", 0, r)][:3]
        assert not slow, "rank %d: the stream was drained after record_frame at steps %r" % (r, slow)
        assert idx == list(range(FRAME_STEPS)), idx
        for step, rec in enumerate(recs):
            assert rec.tobytes() == want_more[step].tobytes(), (r, step, rec, want_more[step])


# ---- the scene's --stats ----------------------------------------------------------------------------------------------
def _plain_scene_rows(res, frames):
    """Frames of the whole-grid jacobi plume, each followed by a synchronous download and the host reduction."""
    mconf = scene.scene_mconf(res, "jacobi")
    zeros = lambda c: torch.zeros(1, c, res, res, res, dtype=torch.float32, device="cuda")   # noqa: E731
    batch = {"pDiv": zeros(1), "UDiv": zeros(3), "flags": torch.from_numpy(scene.scene_flags(res)).cuda(),
             "density": zeros(1)}
    simulate.createPlumeBCs(batch, scene.DENSITY_VAL, 1.0 * (res / 128), scene.PLUME_RAD)
    orc, rows = oracle.Oracle(), []
    for i in range(1, frames + 1):
        simulate.simulate_fused(None, mconf, batch)
        r = ref.record(orc, batch["UDiv"].cpu().numpy(), batch["flags"].cpu().numpy())
        rows.append((i, r[0, 0], r[0, 1], r[0, 2] * mconf["dt"]))
    return rows


def test_scene_stats_equal_a_plain_loop(tmp_path):
    res, frames = 32, 12
    want = _plain_scene_rows(res, frames)
    logs = []
    for slabs in (False, True):
        path = os.path.join(str(tmp_path), "stats_%d.csv" % slabs)
        out = scene.run(res, "plume", "jacobi", num_frames=frames, out_dir=str(tmp_path / ("o%d" % slabs)),
                        log=logs.append, slabs=slabs, world=1, rank=0, stats=path)
        got = scene.read_stats(path)
        assert got == want, (slabs, got[:2], want[:2])
        assert out["max_u_dt"] == max(r[3] for r in want)
    assert any("largest max|U| dt" in m and "--margin" in m for m in logs), logs
