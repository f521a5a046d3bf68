"""Measurement script (not a test): what banked projection networks cost on z-slabs, on one GPU.
  1. the world-1 library slab step (tfl_slab_sim_step) against tfl_simulate_step with the same banked model, at
     n^3 for n in SIZES, banksNum 2 and 3 ('concat', 3xTF32);
  2. one interior rank's workload of an 8-way 256^3 decomposition (the technique of dbg_slab_rank.py: no
     communicator, the exchanges are skipped and the ghost planes go stale): single-bank at margin 2 against banksNum
     2 and 3 at their smallest margins (tfl_slab_cnn_margin) -- the per-rank price of the wider halo.
Prints the card's name and power limit first.  usage: dbg_slab_banks.py [steps]"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from fluidnet_b200 import model as fmodel, simulate, synth, tfluids  # noqa: E402
from fluidnet_b200.slab import cnn_margin  # noqa: E402

STEPS = int(sys.argv[1]) if len(sys.argv) > 1 else 20
SIZES = (128, 256)


def banks(n):
    return None if n == 1 else {"num": n, "split_stage": 1, "join_stage": 3, "aggregate": "concat"}


def timed(step, steps=STEPS, warm=3):
    for _ in range(warm):
        step()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        step()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def slab_sim(ctx, batch_np, n, margin, rank, world):
    lib = ctx.lib
    ctx.check(lib.tfl_comm_init(ctx.h, None, rank, world))      # nil id: rank / world without a communicator
    host = lambda k: np.ascontiguousarray(batch_np[k], np.float32)
    arrs = [host(k) for k in ("flags", "UBC", "UBCInvMask", "densityBC", "densityBCInvMask")]
    h = C.c_void_p()
    ctx.use_current_stream()
    ctx.check(lib.tfl_slab_sim_create(ctx.h, n, n, n, margin, *[a.ctypes.data for a in arrs], C.byref(h)))
    ctx.check(lib.tfl_slab_sim_upload(ctx.h, h, host("pDiv").ctypes.data, host("UDiv").ctypes.data,
                                      host("density").ctypes.data))
    return h


def main():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    print("card: %s" % (q[0] if q else "unknown"))
    ctx = tfluids.context(0)
    lib = ctx.lib
    print("1. world-1 library slab step vs tfl_simulate_step (ms / step, %d steps)" % STEPS)
    for n in SIZES:
        batch_np, mconf, _ = bench.make_problem(n)
        mc = simulate.make_mconf(mconf)
        for nb in (2, 3):
            gm = fmodel.ProjectionModel(synth.make_model(True, banks=banks(nb))["layers"], True, banks=banks(nb))
            gb = {k: torch.from_numpy(v.copy()).cuda() for k, v in batch_np.items()}
            t_fused = timed(lambda: simulate.simulate_fused(None, mconf, gb, gm))
            h = slab_sim(ctx, batch_np, n, cnn_margin(nb), 0, 1)
            t_slab = timed(lambda: ctx.check(lib.tfl_slab_sim_step(ctx.h, h, C.byref(mc), gm.h)))
            lib.tfl_slab_sim_destroy(ctx.h, h)
            lib.tfl_comm_destroy(ctx.h)
            print("  %d^3 banksNum %d: tfl_simulate_step %.3f  slab step (world 1, margin %d) %.3f  ratio %.3f"
                  % (n, nb, t_fused, cnn_margin(nb), t_slab, t_slab / t_fused))
            del gm, gb
    n, world, rank = 256, 8, 3
    print("2. rank %d of an %d-way %d^3 decomposition, exchanges skipped (ms / step, %d steps)" % (rank, world, n, STEPS))
    batch_np, mconf, mnp = bench.make_problem(n)
    mc = simulate.make_mconf(mconf)
    base = None
    for nb in (1, 2, 3):
        layers = mnp["layers"] if nb == 1 else synth.make_model(True, banks=banks(nb))["layers"]
        gm = fmodel.ProjectionModel(layers, True, banks=banks(nb))
        margin = cnn_margin(nb)
        h = slab_sim(ctx, batch_np, n, margin, rank, world)
        info = (C.c_int32 * 6)()
        lib.tfl_slab_sim_layout(h, None, info)
        t = timed(lambda: ctx.check(lib.tfl_slab_sim_step(ctx.h, h, C.byref(mc), gm.h)))
        ctx.trace_faults()       # stale ghost planes may trip the trace guard; the timing is what is wanted
        lib.tfl_slab_sim_destroy(ctx.h, h)
        lib.tfl_comm_destroy(ctx.h)
        base = base or t
        print("  banksNum %d, margin %d (halo %d, %d local planes for %d owned): %.3f ms  (x%.2f of single-bank)"
              % (nb, margin, 2 * margin + 2, info[1], info[5] - info[4], t, t / base))
        del gm


if __name__ == "__main__":
    main()
