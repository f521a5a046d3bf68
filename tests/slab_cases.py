"""Shared pieces of the z-slab tests: the plume problems of the convnet, banked and Jacobi steps with their
single-GPU references, the spawned ranks and their results, the emulated communicator, and refusals that launch
nothing."""
import os
import socket

import torch
import torch.distributed as dist

from scenes import plume_batch, step_mconf


def free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def collect(procs, q, timeout_s):
    """Results of all ranks; if one rank fails (or time runs out) the others are killed instead of
    being left to hang in a collective."""
    import queue
    import time
    res, t0 = [], time.time()
    while len(res) < len(procs) and time.time() - t0 < timeout_s:
        try:
            r = q.get(timeout=1.0)
            res.append(r)
            if r[1] != "ok":
                break
        except queue.Empty:
            if any(p.exitcode not in (None, 0) for p in procs):
                break
    for p in procs:
        p.join(5 if len(res) == len(procs) else 0.1)
        if p.is_alive():
            p.kill()
    return res


def convnet_problem(n):
    from fluidnet_b200 import synth
    return plume_batch(n, inflow=n / 128.0 * 4), step_mconf(n), synth.make_model(True)


def slab_worker(rank, world, port, n, steps, q, native=False, peer=True):
    try:
        os.environ["MASTER_ADDR"] = "127.0.0.1"
        os.environ["MASTER_PORT"] = str(port)
        torch.cuda.set_device(rank)
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
        from fluidnet_b200 import simulate, model as fmodel
        from fluidnet_b200.slab import SlabSimulator, NativeSlabSimulator
        batch, mconf, mnp = convnet_problem(n)
        tb = {k: torch.from_numpy(v) for k, v in batch.items()}
        kw = {"peer_halos": peer} if native else {}
        sim = (NativeSlabSimulator if native else SlabSimulator)(tb, mconf, mnp["layers"], torch.device("cuda", rank),
                                                               rank, world, **kw)
        if native and peer:
            assert sim.halo_transport.startswith("peer memory"), sim.halo_transport
        for _ in range(steps):
            sim.step()
        sim.check()
        got = {k: sim.gather(k) for k in ("density", "UDiv", "pDiv")}
        if rank == 0:
            gb = {k: v.cuda() for k, v in tb.items()}
            gm = fmodel.ProjectionModel(mnp["layers"], True)
            for _ in range(steps):
                simulate.simulate(None, mconf, gb, gm)
            for k in ("density", "UDiv", "pDiv"):
                want = gb[k].cpu()
                err = (got[k] - want).abs().max().item()
                scale = max(want.abs().max().item(), 1e-6)
                assert err <= 1e-6 * scale, "%s: %g vs scale %g" % (k, err, scale)
            # advected density never went through the reduction: bit-exact after one step? after
            # `steps` steps it has seen the projected velocity, so only the tolerance above applies.
        dist.barrier()
        dist.destroy_process_group()
        q.put((rank, "ok"))
    except Exception as e:       # pragma: no cover
        import traceback
        q.put((rank, "FAIL: %s" % traceback.format_exc()))
        raise


BANKED_TOL = {"tf32x3": 1e-6, "tf32": 3e-3}


def banked_problem(gnz, ny, nx, bk):
    from fluidnet_b200 import synth
    batch = plume_batch((gnz, ny, nx), inflow=nx / 128.0 * 4)
    return {k: torch.from_numpy(v) for k, v in batch.items()}, step_mconf(nx), synth.make_model(True, banks=bk)


def single_gpu(tb, mconf, mnp, bk, mode, fused=False):
    from fluidnet_b200 import simulate, model as fmodel
    gb = {k: v.cuda() for k, v in tb.items()}
    gm = fmodel.ProjectionModel(mnp["layers"], True, banks=bk)
    gm.set_mode(mode)
    return gb, lambda: (simulate.simulate_fused if fused else simulate.simulate)(None, mconf, gb, gm)


def refused(ctx, call):
    before = ctx.lib.tfl_launch_count(ctx.h)
    rc = call()
    msg = ctx.lib.tfl_last_error(ctx.h)
    assert rc != 0 and b"z-slab" in msg, msg
    assert ctx.lib.tfl_launch_count(ctx.h) == before, "a refused call launched work"
    return msg


def jacobi_problem(nx, ny, gnz, buoyancy=True, gravity=False, vorticity=True, max_iter=34, seed=7):
    batch = plume_batch((gnz, ny, nx), flags_seed=seed, inflow=max(nx, gnz) / 128.0 * 4)
    over = {} if buoyancy else {"buoyancyScale": 0.0}
    mconf = step_mconf(nx, gravityScale=0.5 if gravity else 0.0, vorticityConfinementAmp=3.0 if vorticity else 0.0,
                       simMethod="jacobi", maxIter=max_iter, **over)
    return {k: torch.from_numpy(v) for k, v in batch.items()}, mconf


def jacobi_reference(tb, mconf, steps):
    """Single-GPU operator sequence, state after each step."""
    from fluidnet_b200 import simulate
    gb = {k: v.cuda() for k, v in tb.items()}
    out = []
    for _ in range(steps):
        simulate.simulate(None, mconf, gb)
        out.append({k: gb[k].cpu().clone() for k in KEYS})
    return out


class Comm:
    """allgather over one queue per rank; every rank calls it the same number of times, in the same order."""

    def __init__(self, rank, world, inboxes):
        self.rank, self.world, self.inboxes, self.n, self.early = rank, world, inboxes, 0, {}

    def allgather(self, obj):
        self.n += 1
        for r, qr in enumerate(self.inboxes):
            if r != self.rank:
                qr.put((self.n, self.rank, obj))
        got = {self.rank: obj}
        while len(got) < self.world:
            key = next((k for k in self.early if k[0] == self.n), None)
            if key is not None:
                got[key[1]] = self.early.pop(key)
                continue
            n, r, o = self.inboxes[self.rank].get(timeout=TIMEOUT_S)
            if n == self.n:
                got[r] = o
            else:                                   # a faster rank's next allgather
                self.early[(n, r)] = o
        return [got[r] for r in range(self.world)]


KEYS = ("pDiv", "UDiv", "density")


TIMEOUT_S = 400
