"""The library's multi-rank z-slab step (tfl_slab_sim_step at world > 1) with one process per rank, every process on
cuda:0 with its own context: the peer-memory halo exchanges (k_slab_push / k_slab_pull), the 2-double all-reduce of
the input scale (k_sum_push / k_sum_pull) and the Jacobi p exchanges, over real CUDA IPC mappings.  The ranks run
NativeSlabSimulator without torch.distributed: no NCCL communicator, the IPC handles go through an allgather over
multiprocessing queues.  Without MPS the processes time-slice the GPU, so a bounded wait on the device ends as soon
as the rank it waits for gets its turn.

One group of processes per world size runs its whole list of cases, a fresh simulator per case (so inboxes are
exported and mapped again within each process).  Every rank downloads its owned planes after every step and sends
them to rank 0, which assembles the global fields and compares them with references it computes itself on cuda:0:

  jacobi   p, U and density equal the single-GPU step bit for bit (worlds 2 - 5, margins 2 and 3, maxIter 1, k - 1,
           k, k + 1, 34, 100 with k = 2 margin + 2, the thinnest legal and uneven slabs, the one-launch block kernel);
  convnet  equal the emulated run (SlabSimulator + run_lockstep at the same world, margin, model and mode) bit for
           bit -- both drivers call the same operators on the same plane ranges and add the partial sums in rank
           order from zero -- and the single-GPU step within test_gpu_slab_banks.py's tolerance;
  traffic  after every step, each rank's exchange_stats / jacobi_stats bytes and count equal what the shapes and the
           Jacobi schedule say: one message per neighbour of width x ny x nx x channels floats;
  skew     a rank that starts each step ~30 ms late (a different rank every step) changes nothing: its neighbours
           push the next exchange while it still scatters the last one;
  frames   SlabFrameRecorder frames of the real step equal the single-GPU density of the same step, in .vbox order.

Every rank reports its fault count per case (must be 0).  All checks run after the case's collective close, so a
failing check never leaves a neighbour waiting on the device."""
import time

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from slab_cases import Comm, TIMEOUT_S, collect

pytestmark = pytest.mark.gpu

KEYS = ("pDiv", "UDiv", "density")
SKEW_S = 0.03                        # far below the ~2 s bound of k_slab_pull / k_sum_pull
FORCES = [(True, False, True), (True, True, False), (False, True, True), (False, False, False)]


def _jacobi(world, nx, ny, gnz, margin, it, forces, steps=3, skew=False, frames=False):
    k = 2 * margin + 2
    iters = {"k-1": k - 1, "k": k, "k+1": k + 1}.get(it, it)
    return dict(kind="jacobi", world=world, shape=(gnz, ny, nx), margin=margin, iters=iters, forces=forces,
                steps=steps, skew=skew, frames=frames, name="jacobi w%d %dx%dx%d m%d it%s %s%s%s" % (
                    world, gnz, ny, nx, margin, iters, "".join("BGV"[i] for i in range(3) if forces[i]) or "-",
                    " skew" if skew else "", " frames" if frames else ""))


def _convnet(world, gnz, ny, nx, bk, mode, steps=3, skew=False):
    return dict(kind="convnet", world=world, shape=(gnz, ny, nx), bk=bk, mode=mode, steps=steps, skew=skew,
                frames=False, name="convnet w%d %dx%dx%d %s %s%s" % (world, gnz, ny, nx, "N%d-%s" % bk if bk else "N1",
                                                                  mode, " skew" if skew else ""))


def _cases(world):
    out = []
    # margin 2 (halo 6): gnz = 6 world + 1, the thinnest legal slabs (6 planes) and an uneven split; nx = 128 grids
    # take the one-launch block kernel, nx = 32 the per-sweep launches
    for i, it in enumerate((1, "k-1", "k", "k+1", 34, 100)):
        nx, ny = (128, 16) if i % 2 else (32, 24)
        out.append(_jacobi(world, nx, ny, 6 * world + 1, 2, it, FORCES[i % 4]))
    # margin 3 (halo 8): 16 over 2 is two thinnest even slabs, the others split unevenly
    gnz = {2: 16, 3: 26, 4: 35, 5: 41}[world]
    out.append(_jacobi(world, 128, 16, gnz, 3, "k+1", FORCES[1]))
    out.append(_jacobi(world, 32, 24, gnz, 3, 34, FORCES[2]))
    # single bank at margin 2: 40 over 3 splits at planes 14 and 27 (odd, uneven); 28 over 4 is four thinnest slabs
    conv = {2: (32, 16, 16), 3: (40, 16, 24), 4: (28, 16, 16)}
    if world in conv:
        for mode in ("tf32x3", "tf32"):
            out.append(_convnet(world, *conv[world], None, mode))
    if world == 3:
        # banked at tfl_slab_cnn_margin: N = 2 (margin 3) split at 14 / 27, N = 3 (margin 6, halo 14) at 15 / 30
        out.append(_convnet(3, 40, 16, 16, (2, "concat"), "tf32x3"))
        out.append(_convnet(3, 44, 16, 16, (3, "add"), "tf32x3"))
        out.append(_jacobi(3, 128, 16, 19, 2, 100, FORCES[0], steps=4, skew=True))
        out.append(_convnet(3, 40, 16, 24, None, "tf32x3", steps=4, skew=True))
        out.append(_jacobi(3, 128, 16, 20, 2, 34, FORCES[2], steps=4, frames=True))
    return out


def _problem(case):
    """Global batch, mconf, model layers (None for 'jacobi') and banks of a case."""
    gnz, ny, nx = case["shape"]
    if case["kind"] == "jacobi":
        from slab_cases import jacobi_problem
        tb, mconf = jacobi_problem(nx, ny, gnz, *case["forces"], max_iter=case["iters"])
        return tb, mconf, None, None
    from scenes import banks
    from slab_cases import banked_problem
    bk = banks(*case["bk"]) if case["bk"] else None
    tb, mconf, mnp = banked_problem(gnz, ny, nx, bk)
    return tb, mconf, mnp["layers"], bk


def _references(case):
    """Per step: the single-GPU state and, for 'convnet', the emulated run's (global CPU tensors)."""
    from slab_cases import jacobi_reference
    tb, mconf, layers, bk = _problem(case)
    if case["kind"] == "jacobi":
        return {"single": jacobi_reference(tb, mconf, case["steps"])}
    from slab_cases import single_gpu
    from fluidnet_b200.slab import SlabSimulator, run_lockstep
    dev = torch.device("cuda", 0)
    sims = [SlabSimulator(tb, mconf, layers, dev, rank=r, world=case["world"], banks=bk, conv_mode=case["mode"])
            for r in range(case["world"])]
    gb, step = single_gpu(tb, mconf, {"layers": layers}, bk, case["mode"])
    emu, single = [], []
    for _ in range(case["steps"]):
        run_lockstep(sims)
        step()
        emu.append({k: torch.cat([q.dec.owned(q.s[k]).cpu() for q in sims], dim=2) for k in KEYS})
        single.append({k: gb[k].cpu().clone() for k in KEYS})
    torch.cuda.synchronize()
    return {"emulated": emu, "single": single}


def _want_traffic(case, rank):
    """(bytes of exchanges 0, 1, 2, p exchanges, p exchange bytes) this rank sends per step."""
    from fluidnet_b200.slab import cnn_margin, jacobi_schedule
    world, (gnz, ny, nx) = case["world"], case["shape"]
    plane = ny * nx
    nbrs = (rank > 0) + (rank < world - 1)
    msg = lambda width, chans: nbrs * width * plane * chans * 4        # noqa: E731  one message per neighbour
    if case["kind"] == "convnet":
        n = case["bk"][0] if case["bk"] else 1
        halo = 2 * cnn_margin(n) + 2
        return [msg(halo, 4), msg(4, 4), msg(2 * cnn_margin(n) + 1, 4)], 0, 0
    margin, iters = case["margin"], case["iters"]
    halo = 2 * margin + 2
    nblk = -(-(iters + 1) // halo)                 # blocks of `halo` sweeps, the last one the rest and one more plane
    widths = [halo] * (nblk - 1) + [iters - (nblk - 1) * halo + 1]
    (_, _, u_width), blocks = jacobi_schedule(gnz, world, rank, margin, iters)
    assert [b[1] for b in blocks] == [0] + widths[1:] and u_width == max(widths), (blocks, widths)
    return [msg(halo, 4), msg(4, 4), msg(u_width, 3)], nblk - 1, msg(sum(widths[1:]), 1)


def _run_case(case, ci, rank, world, comm, barrier, qd):
    """One case on this rank; returns (traffic per step, frames (rank 0), fault count)."""
    from fluidnet_b200.slab import NativeSlabSimulator
    tb, mconf, layers, bk = _problem(case)
    sim = NativeSlabSimulator(tb, mconf, layers, torch.device("cuda", 0), rank, world,
                              margin=case.get("margin"), banks=bk, conv_mode=case.get("mode"),
                              allgather=comm.allgather, barrier=barrier)
    assert sim.halo_transport.startswith("peer memory"), sim.halo_transport
    rec = sim.frame_recorder(slots=2) if case["frames"] else None
    traffic, frames = [], []
    for step in range(case["steps"]):
        if case["skew"] and rank == step % world:
            time.sleep(SKEW_S)
        sim.step()
        if rec is not None:
            sim.record(rec, None)
            if rank == 0:
                idx, frame = rec.take(wait=True)
                frames.append((idx, frame.view(np.uint32).copy()))
                rec.release()
        by = sim.exchange_stats()[1]
        n, _, jby = sim.jacobi_stats()
        traffic.append((by, n, jby))
        d = sim.download()
        qd.put((ci, step, rank, sim.z0, sim.z1, {k: d[k][:, :, sim.z0:sim.z1].copy() for k in KEYS}))
    torch.cuda.synchronize()
    faults = sim.ctx.trace_faults()
    if rec is not None:
        rec.close()
    sim.close()                            # synchronise, barrier, destroy, barrier
    return traffic, frames, faults


def _first_diff(got, want):
    """First global plane (and channel) where two [1][c][z][y][x] tensors differ, and the largest difference."""
    ne = (got != want) & ~(torch.isnan(got) & torch.isnan(want))
    z = ne.any(dim=4).any(dim=3).any(dim=1)[0].nonzero()
    c = ne.any(dim=4).any(dim=3).any(dim=2)[0].nonzero()
    return "first plane z=%d (channel %d), max |diff| %g" % (int(z[0]), int(c[0]), (got - want).abs().max().item())


def _check_case(case, refs, parts, frames):
    """Rank 0: compares the assembled fields of every step; returns failure strings."""
    fails = []
    gnz, ny, nx = case["shape"]
    for step in range(case["steps"]):
        got = {}
        for k in KEYS:
            c = 3 if k == "UDiv" else 1
            a = torch.full((1, c, gnz, ny, nx), float("nan"))
            for z0, z1, arr in parts[step]:
                a[:, :, z0:z1] = torch.from_numpy(arr[k])
            got[k] = a
        for k in KEYS:
            what = "%s: step %d %s" % (case["name"], step, k)
            if case["kind"] == "jacobi":
                want = refs["single"][step][k]
                if not torch.equal(got[k], want):
                    fails.append("%s differs from the single-GPU step: %s" % (what, _first_diff(got[k], want)))
                continue
            emu, single = refs["emulated"][step][k], refs["single"][step][k]
            if not torch.equal(got[k], emu):
                fails.append("%s differs from the emulated run: %s" % (what, _first_diff(got[k], emu)))
            from slab_cases import BANKED_TOL
            err = (got[k] - single).abs().max().item()
            scale = max(single.abs().max().item(), 1e-6)
            if not err <= BANKED_TOL[case["mode"]] * scale:
                fails.append("%s: %g from the single-GPU step (scale %g)" % (what, err, scale))
    if case["frames"]:
        if [i for i, _ in frames] != list(range(case["steps"])):
            fails.append("%s: frame indices %r" % (case["name"], [i for i, _ in frames]))
        for step, (_, frame) in enumerate(frames):
            want = refs["single"][step]["density"].numpy()[0, 0].transpose(2, 1, 0)
            if not (frame.shape == want.shape and np.array_equal(frame, want.view(np.uint32))):
                fails.append("%s: frame %d is not the single-GPU density" % (case["name"], step))
    return fails


def _worker(rank, world, q, qd, inboxes, barrier):
    try:
        torch.cuda.set_device(0)
        comm = Comm(rank, world, inboxes)
        wait = lambda: barrier.wait(TIMEOUT_S)       # noqa: E731
        fails, compared, pending = [], 0, {}
        for ci, case in enumerate(_cases(world)):
            refs = _references(case) if rank == 0 else None
            traffic, frames, faults = _run_case(case, ci, rank, world, comm, wait, qd)
            if faults:
                fails.append("%s: rank %d counted %d faults" % (case["name"], rank, faults))
            want = _want_traffic(case, rank)
            for step, got in enumerate(traffic):
                if got != (want[0], want[1], want[2]):
                    fails.append("%s: rank %d step %d sent (bytes of exchanges 0-2, p exchanges, p bytes) %r, the "
                                 "shapes and the schedule say %r" % (case["name"], rank, step, got, want))
            if rank == 0:
                while len([k for k in pending if k[0] == ci]) < world * case["steps"]:
                    c, step, r, z0, z1, arrs = qd.get(timeout=TIMEOUT_S)
                    pending[(c, step, r)] = (z0, z1, arrs)
                parts = [[pending.pop((ci, s, r)) for r in range(world)] for s in range(case["steps"])]
                fails += _check_case(case, refs, parts, frames)
                compared += case["steps"]
        q.put((rank, "ok", fails, compared))
    except Exception:               # pragma: no cover
        import traceback
        q.put((rank, "FAIL: %s" % traceback.format_exc(), [], 0))
        raise


@pytest.mark.parametrize("world", [2, 3, 4, 5])
def test_library_step_one_process_per_rank(world):
    """world processes on cuda:0 run every case of _cases(world) through tfl_slab_sim_step over peer memory."""
    ctx = mp.get_context("spawn")
    q, qd, barrier = ctx.Queue(), ctx.Queue(), ctx.Barrier(world)
    inboxes = [ctx.Queue() for _ in range(world)]
    procs = [ctx.Process(target=_worker, args=(r, world, q, qd, inboxes, barrier)) for r in range(world)]
    for p in procs:
        p.start()
    res = collect(procs, q, TIMEOUT_S)
    assert len(res) == world and all(r[1] == "ok" for r in res), res
    fails = [f for r in res for f in r[2]]
    assert not fails, "\n".join(fails)
    assert sum(r[3] for r in res) == sum(c["steps"] for c in _cases(world))


def test_missing_peer_refuses_before_any_step():
    """Without torch.distributed there is no NCCL to fall back on: a rank whose peer reports no inbox raises, by name,
    before anything is launched, and leaves the context at one rank without a communicator."""
    from fluidnet_b200._lib import TflError
    from fluidnet_b200.slab import NativeSlabSimulator
    from slab_cases import jacobi_problem
    tb, mconf = jacobi_problem(32, 24, 16, max_iter=5)
    dev = torch.device("cuda", 0)
    gathered = []

    def allgather(obj):
        gathered.append(obj)
        return [obj, None]                                  # rank 1's handle is missing

    for bad in (dict(allgather=allgather), dict(barrier=lambda: None)):
        with pytest.raises(ValueError, match="together"):
            NativeSlabSimulator(tb, mconf, None, dev, rank=0, world=2, **bad)
    with pytest.raises(ValueError, match="peer memory"):
        NativeSlabSimulator(tb, mconf, None, dev, rank=0, world=2, peer_halos=False, allgather=allgather,
                            barrier=lambda: None)
    from fluidnet_b200 import tfluids
    ctx = tfluids.context(dev)
    l0 = ctx.launch_count()
    with pytest.raises(TflError, match=r"rank 1: no inbox handle.*no NCCL fallback"):
        NativeSlabSimulator(tb, mconf, None, dev, rank=0, world=2, allgather=allgather, barrier=lambda: None)
    assert ctx.launch_count() == l0
    assert len(gathered) == 1 and isinstance(gathered[0], bytes)       # rank 0 did export its inbox
    # the context is back at one rank: a world-1 simulator without torch.distributed steps as before
    sim = NativeSlabSimulator(tb, mconf, None, dev, rank=0, world=1, allgather=allgather, barrier=lambda: None)
    sim.step()
    sim.check()
    assert torch.equal(sim.gather("density"), torch.from_numpy(sim.download()["density"]))
    sim.close()
