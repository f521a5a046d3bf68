"""Timing script (not a test): the world-1 z-slab step with simMethod 'jacobi' solved to pTol 1e-5 (maxIter 2000) on
the plume's first step at 64^3, 128^3 and 256^3, each timed from the same state (uploaded again before every round):

  direct    tfl_slab_sim_step with the tolerance (waits once per chunk of blocks)
  replay    the same step replayed from a slab graph (the loop runs on the device)
  whole     the whole-grid operator sequence with solveLinearSystemJacobiDevice as its solve
  fixed     the fixed-count slab step (pTol 0) with maxIter = the sweeps the tolerance step ran
  stop      direct and replayed again with a pTol that stops the solve on the first sweep of a block (sweep 1002): the
            block runs again up to it, and the rest of the chunk's blocks are gated no-ops

Every variant ends in a device synchronise; the median of --rounds rounds is kept.  Prints the GPU's name and power
limit beside the numbers, and one JSON line.

    python tests/dbg_slab_jacobi_tol.py [--sizes 64,128,256] [--rounds 5]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from slab_cases import jacobi_problem                  # noqa: E402

TOL, MAX_ITER = 1e-5, 2000
STOP_PROBE = 1002


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return r.stdout.strip().splitlines()[torch.cuda.current_device()] if r.returncode == 0 else "unknown"


def timed(fn, before, rounds):
    ts = []
    for _ in range(rounds + 1):                        # the first round warms up
        before()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return sorted(ts[1:])[rounds // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="64,128,256")
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    from fluidnet_b200 import simulate, tfluids
    from fluidnet_b200.slab import NativeSlabSimulator, SlabStepGraph
    info = gpu_info()
    print("GPU:", info)
    rows = []
    stream = torch.cuda.Stream()
    for n in [int(v) for v in args.sizes.split(",")]:
        tb, mconf = jacobi_problem(n, n, n, max_iter=MAX_ITER)
        host = {k: v.numpy().copy() for k, v in tb.items()}
        with torch.cuda.stream(stream):
            sim = NativeSlabSimulator(tb, mconf, None, torch.device("cuda", 0), rank=0, world=1)

            def reset(s=sim):
                s.ctx.check(s.ctx.lib.tfl_slab_sim_upload(s.ctx.h, s.h, host["pDiv"].ctypes.data,
                                                          host["UDiv"].ctypes.data, host["density"].ctypes.data))
            sim.set_jacobi_tolerance(TOL)
            reset()
            sim.step()
            res, iters = sim.jacobi_status()
            sweeps = iters + 1 if res < TOL else iters      # a stop on res < pTol does not count its sweep
            direct = timed(sim.step, reset, args.rounds)
            graph = SlabStepGraph(sim)
            replay = timed(graph.launch, reset, args.rounds)
            graph.close()
            # a solve that stops: pTol just above the residual of sweep 1002 (the first of a block of 6), so the
            # stopping block runs again up to it and a chunk of gated blocks follows the stop
            sim.set_jacobi_tolerance(1e-30)
            sim.mc.max_iter = STOP_PROBE + 1
            reset()
            sim.step()
            sim.set_jacobi_tolerance(sim.jacobi_status()[0] * (1 + 1e-6))
            sim.mc.max_iter = MAX_ITER
            reset()
            sim.step()
            s_res, s_iters = sim.jacobi_status()
            s_direct = timed(sim.step, reset, args.rounds)
            graph = SlabStepGraph(sim)
            s_replay = timed(graph.launch, reset, args.rounds)
            graph.close()
            sim.set_jacobi_tolerance(0.0)
            sim.mc.max_iter = sweeps
            fixed = timed(sim.step, reset, args.rounds)
            sim.close()
        orig = tfluids.solveLinearSystemJacobi

        def dev_solve(p, flags, div, is3D, pTol=None, maxIter=None, verbose=None):
            tfluids.solveLinearSystemJacobiDevice(p, flags, div, is3D, TOL, maxIter)
        gb = {}

        def fresh():
            gb.update({k: v.cuda() for k, v in tb.items()})
        tfluids.solveLinearSystemJacobi = dev_solve
        try:
            whole = timed(lambda: simulate.simulate(None, mconf, gb), fresh, args.rounds)
        finally:
            tfluids.solveLinearSystemJacobi = orig
        row = dict(n=n, iterations=iters, sweeps=sweeps, residual=res, direct_ms=direct, replay_ms=replay,
                   whole_grid_dev_ms=whole, fixed_ms=fixed, tol_us_per_sweep=1e3 * direct / sweeps,
                   fixed_us_per_sweep=1e3 * fixed / sweeps, stop_iterations=s_iters, stop_direct_ms=s_direct,
                   stop_replay_ms=s_replay)
        rows.append(row)
        print("%4d^3  %5d sweeps  direct %8.2f ms  replay %8.2f ms  whole-grid _dev %8.2f ms  fixed %8.2f ms  "
              "(%.2f / %.2f us per sweep)" % (n, sweeps, direct, replay, whole, fixed, row["tol_us_per_sweep"],
                                              row["fixed_us_per_sweep"]))
        print("        stop after sweep %d (residual %.6g): direct %8.2f ms  replay %8.2f ms" % (s_iters, s_res, s_direct,
                                                                                             s_replay))
    print(json.dumps({"gpu": info, "p_tol": TOL, "max_iter": MAX_ITER, "rows": rows}))


if __name__ == "__main__":
    main()
