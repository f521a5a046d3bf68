"""The z-slab step replayed from a CUDA graph (tfl_slab_graph_*, slab.SlabStepGraph): one tfl_slab_sim_step captured
on the context's stream and replayed with one launch, its exchanges' sequence numbers read and advanced on the device.

  world 1   in one process: convnet N = 1 in 3xTF32 and TF32, banked N = 2 'concat', Jacobi at maxIter 34 on nx = 128
            (the cooperative block kernel) and nx = 32 (one launch per sweep).  One direct step, then replays, and a
            sequence that interleaves direct steps and replays: p, U and density equal an all-direct run bit for bit
            after every one of 12 steps, no fault is counted, and a replay adds to tfl_launch_count what a direct step
            adds.
  ranks     one process per rank on cuda:0 (worlds 2 - 4, the peer-memory exchanges over real CUDA IPC mappings, as in
            test_gpu_slab_ranks.py; Jacobi and the single-bank model at every world, the banked model at worlds 2 and
            3): every case runs twice in the same processes, once with direct steps only and once
            with replays -- all ranks replaying after the first step, ranks mixing direct steps and replays on
            different steps, a rank starting each replay ~30 ms late.  Each rank's owned planes, its exchange bytes and
            p-exchange counts, the SlabFrameRecorder frames and the monitor records taken between steps must equal the
            direct run's bit for bit.
  refusals  the default stream, no earlier direct step, simMethod 'pcg', a model the slab step refuses, and a graph
            made stale by the model running on another grid: each launches nothing and names its cause.  The refusal
            of the NCCL transport at world > 1 cannot be reached here: NCCL needs one GPU per rank, and this test has
            one GPU.
"""
import ctypes as C
import time

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from slab_cases import Comm, KEYS, TIMEOUT_S, collect

pytestmark = pytest.mark.gpu

SKEW_S = 0.03                        # far below the ~2 s bound of k_slab_pull / k_sum_pull


def _problem(case):
    """Global batch, mconf, model layers (None for 'jacobi'), banks and conv mode of a case."""
    gnz, ny, nx = case["shape"]
    if case["kind"] == "jacobi":
        from slab_cases import jacobi_problem
        tb, mconf = jacobi_problem(nx, ny, gnz, max_iter=34)
        return tb, mconf, None, None, None
    from scenes import banks
    from slab_cases import banked_problem
    bk = banks(*case["bk"]) if case.get("bk") else None
    tb, mconf, mnp = banked_problem(gnz, ny, nx, bk)
    return tb, mconf, mnp["layers"], bk, case["mode"]


def _sim(case, rank=0, world=1, **kw):
    from fluidnet_b200.slab import NativeSlabSimulator
    tb, mconf, layers, bk, mode = _problem(case)
    return NativeSlabSimulator(tb, mconf, layers, torch.device("cuda", 0), rank, world, banks=bk, conv_mode=mode, **kw)


def _fields(sim):
    d = sim.download()
    return {k: d[k][:, :, sim.z0:sim.z1].copy() for k in KEYS}


def _differ(a, b):
    return [k for k in KEYS if not np.array_equal(a[k].view(np.uint32), b[k].view(np.uint32))]


# ---- world 1, in process ----------------------------------------------------------------------------------------------

WORLD1 = {
    "convnet N1 tf32x3": dict(kind="convnet", shape=(32, 32, 32), mode="tf32x3"),
    "convnet N1 tf32": dict(kind="convnet", shape=(32, 32, 32), mode="tf32"),
    "banked N2 concat": dict(kind="convnet", shape=(32, 32, 32), bk=(2, "concat"), mode="tf32x3"),
    "jacobi nx128 block": dict(kind="jacobi", shape=(24, 16, 128)),
    "jacobi nx32 per-sweep": dict(kind="jacobi", shape=(24, 24, 32)),
}
STEPS = 12
MIXED = "DRRDRDDRRRDR"                 # D: direct step, R: replay (the first step is always direct)


@pytest.mark.parametrize("name", sorted(WORLD1))
def test_world1_replays_equal_direct_steps(name):
    from fluidnet_b200.slab import SlabStepGraph
    case = WORLD1[name]
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        direct, replayed, mixed = _sim(case), _sim(case), _sim(case)
        ctx = direct.ctx
        ctx.trace_faults()
        graphs = {}
        try:
            for step in range(STEPS):
                l0 = ctx.launch_count()
                direct.step()
                per_direct = ctx.launch_count() - l0
                for key, sim, how in (("all", replayed, "R"), ("mixed", mixed, MIXED[step])):
                    l0 = ctx.launch_count()
                    if step == 0 or how == "D":
                        sim.step()
                    else:
                        graphs[key].launch()
                    got = ctx.launch_count() - l0
                    assert got == per_direct, "%s step %d (%s): %d launches counted, a direct step %d" % (
                        key, step, how, got, per_direct)
                    if step == 0:
                        graphs[key] = SlabStepGraph(sim)
                want = _fields(direct)
                for key, sim in (("all", replayed), ("mixed", mixed)):
                    bad = _differ(_fields(sim), want)
                    assert not bad, "%s: %s after step %d (%s) differ from the direct run" % (
                        name, bad, step, key)
            stream.synchronize()
            assert ctx.trace_faults() == 0
        finally:
            for g in graphs.values():
                g.close()
            for sim in (direct, replayed, mixed):
                sim.close()


# ---- refusals ---------------------------------------------------------------------------------------------------------

def _refused(ctx, call, *words):
    from fluidnet_b200._lib import TflError
    before = ctx.launch_count()
    with pytest.raises(TflError) as e:
        call()
    msg = str(e.value)
    assert msg.startswith("slab_graph") and all(w in msg for w in words), msg
    assert ctx.launch_count() == before, "a refused call launched work"
    return msg


def test_refusals_launch_nothing_and_name_their_cause():
    from fluidnet_b200 import simulate
    from fluidnet_b200.slab import SlabStepGraph
    conv = WORLD1["convnet N1 tf32x3"]
    # the default stream
    sim = _sim(conv)
    try:
        sim.step()
        _refused(sim.ctx, lambda: SlabStepGraph(sim), "default stream")
    finally:
        sim.close()
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        sim = _sim(conv)
        ctx, lib = sim.ctx, sim.ctx.lib
        graph = None
        try:
            # no earlier direct step
            _refused(ctx, lambda: SlabStepGraph(sim), "no earlier tfl_slab_sim_step")
            sim.step()
            # simMethod 'pcg', with the slab step's own message
            mc = simulate.make_mconf(dict(sim.mconf, simMethod="pcg"))
            h = C.c_void_p()
            _refused(ctx, lambda: ctx.check(lib.tfl_slab_graph_create(ctx.h, sim.h, C.byref(mc), sim.model.h,
                                                                      C.byref(h))), "'pcg' is not decomposed")
            # a model the slab step refuses (the fp32 path)
            sim.model.set_mode("fp32")
            _refused(ctx, lambda: SlabStepGraph(sim), "z-slab", "tensor-core")
            sim.model.set_mode("tf32x3")
            # a graph made stale by the model running on another grid
            graph = SlabStepGraph(sim)
            graph.launch()
            stream.synchronize()
            from scenes import plume_batch, to_gpu
            other = to_gpu(plume_batch(16))
            sim.model.forward((other["pDiv"], other["UDiv"], other["flags"]))
            _refused(ctx, graph.launch, "stale graph", "the model's activation buffers")
            stream.synchronize()
            assert ctx.trace_faults() == 0
        finally:
            if graph is not None:
                graph.close()
            sim.close()


# ---- one process per rank ---------------------------------------------------------------------------------------------

def _cases(world):
    conv = {2: (32, 16, 16), 3: (40, 16, 24), 4: (28, 16, 16)}[world]
    gnz = 6 * world + 1                                   # margin 2: the thinnest legal slabs, split unevenly
    out = [
        dict(name="jacobi nx128 replay", kind="jacobi", shape=(gnz, 16, 128), how="replay"),
        dict(name="jacobi nx32 mixed frames monitor", kind="jacobi", shape=(gnz, 24, 32), how="mixed", frames=True,
             monitor=True),
        dict(name="convnet N1 replay monitor", kind="convnet", shape=conv, mode="tf32x3", how="replay", monitor=True),
        dict(name="convnet N1 replay skew", kind="convnet", shape=conv, mode="tf32x3", how="replay", skew=True),
    ]
    # The banked model at worlds 2 and 3 (margin 3, the split of test_gpu_slab_ranks.py at 3).  At world 4 two runs of
    # the direct step alone on the same inputs already differ in their bits, so there is no direct run to hold a replay
    # to there.
    if world in (2, 3):
        banked = {2: (32, 16, 16), 3: (40, 16, 16)}[world]
        out.append(dict(name="banked N2 mixed", kind="convnet", shape=banked, bk=(2, "concat"), mode="tf32x3",
                        how="mixed"))
    return out


RANK_STEPS = 6


def _replays(how, rank, step):
    """Whether this rank replays step `step` (0-based) in a run of kind `how`."""
    if how == "direct" or step == 0:
        return False
    if how == "mixed":                         # rank r replays every other step, ranks out of phase
        return (step + rank) % 2 == 1
    return True


def _run(case, how, rank, world, comm, barrier):
    """One pass of a case on this rank -> per step: (owned fields, exchange bytes, p exchanges, p bytes), frames
    (rank 0), monitor records, fault count."""
    from fluidnet_b200.slab import SlabStepGraph
    sim = _sim(case, rank, world, allgather=comm.allgather, barrier=barrier)
    assert sim.halo_transport.startswith("peer memory"), sim.halo_transport
    sim.ctx.trace_faults()
    rec = sim.frame_recorder(slots=2) if case.get("frames") else None
    mon = sim.monitor(RANK_STEPS) if case.get("monitor") else None
    graph, out, frames = None, [], []
    try:
        for step in range(RANK_STEPS):
            if case.get("skew") and rank == step % world:
                time.sleep(SKEW_S)
            if _replays(how, rank, step):
                graph.launch()
            else:
                sim.step()
            if graph is None and how != "direct":
                graph = SlabStepGraph(sim)
            if rec is not None:
                sim.record(rec, None)
                if rank == 0:
                    idx, frame = rec.take(wait=True)
                    frames.append((idx, frame.view(np.uint32).copy()))
                    rec.release()
            if mon is not None:
                mon.record()
            by = sim.exchange_stats()[1]
            n, _, jby = sim.jacobi_stats()
            out.append((_fields(sim), (tuple(by), n, jby)))
        records = mon.collect() if mon is not None else []
        torch.cuda.synchronize()
        faults = sim.ctx.trace_faults()
    finally:
        if graph is not None:
            graph.close()
        if mon is not None:
            mon.close()
        if rec is not None:
            rec.close()
        sim.close()                            # synchronise, barrier, destroy, barrier
    return out, frames, [(i, np.asarray(v).copy()) for i, v in records], faults


def _compare(case, how, rank, direct, replay):
    fails = []
    (d_steps, d_frames, d_recs, d_faults), (r_steps, r_frames, r_recs, r_faults) = direct, replay
    what = "%s (%s), rank %d" % (case["name"], how, rank)
    for f, tag in ((d_faults, "direct"), (r_faults, how)):
        if f:
            fails.append("%s: %d faults in the %s run" % (what, f, tag))
    for step, ((df, dt), (rf, rt)) in enumerate(zip(d_steps, r_steps)):
        bad = _differ(rf, df)
        if bad:
            fails.append("%s: %s of step %d differ from the direct run" % (what, bad, step))
        if rt != dt:
            fails.append("%s: step %d traffic (bytes of exchanges 0-2, p exchanges, p bytes) %r, direct %r"
                         % (what, step, rt, dt))
    if len(r_frames) != len(d_frames) or any(i != j or not np.array_equal(a, b)
                                             for (i, a), (j, b) in zip(r_frames, d_frames)):
        fails.append("%s: recorder frames differ from the direct run's" % what)
    if len(r_recs) != len(d_recs) or any(i != j or not np.array_equal(a, b) for (i, a), (j, b) in zip(r_recs, d_recs)):
        fails.append("%s: monitor records differ from the direct run's" % what)
    return fails


def _worker(rank, world, q, inboxes, barrier):
    try:
        torch.cuda.set_device(0)
        comm = Comm(rank, world, inboxes)
        wait = lambda: barrier.wait(TIMEOUT_S)       # noqa: E731
        stream = torch.cuda.Stream()
        fails, compared = [], 0
        with torch.cuda.stream(stream):
            for case in _cases(world):
                direct = _run(case, "direct", rank, world, comm, wait)
                replay = _run(case, case["how"], rank, world, comm, wait)
                fails += _compare(case, case["how"], rank, direct, replay)
                compared += RANK_STEPS
        q.put((rank, "ok", fails, compared))
    except Exception:               # pragma: no cover
        import traceback
        q.put((rank, "FAIL: %s" % traceback.format_exc(), [], 0))
        raise


@pytest.mark.parametrize("world", [2, 3, 4])
def test_replays_equal_direct_steps_one_process_per_rank(world):
    ctx = mp.get_context("spawn")
    q, barrier = ctx.Queue(), ctx.Barrier(world)
    inboxes = [ctx.Queue() for _ in range(world)]
    procs = [ctx.Process(target=_worker, args=(r, world, q, inboxes, barrier)) for r in range(world)]
    for p in procs:
        p.start()
    res = collect(procs, q, TIMEOUT_S)
    assert len(res) == world and all(r[1] == "ok" for r in res), res
    fails = [f for r in res for f in r[2]]
    assert not fails, "\n".join(fails)
    assert sum(r[3] for r in res) == world * RANK_STEPS * len(_cases(world))
