"""Timing of simMethod 'jacobi' on z-slabs at one rank (one GPU): the slab step against tfl_simulate_step, and one block
of sweeps in the one-launch kernel (k_jacobi_resident<KZ>) against one launch per sweep and the single-GPU solve
(the same kernel for maxIter - 1 sweeps plus one k_jacobi_iter4, or k_jacobi_march).  CUDA events, median of --reps
after --warmup.  Prints one JSON line per row.

    python tests/dbg_slab_jacobi.py [--reps 20] [--warmup 5]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _time(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b))
    return statistics.median(out)


def _problem(n, max_iter):
    from fluidnet_b200 import synth
    flags = synth.make_flags(n, n, n, True, nb=1, geometry=True)
    U = synth.make_smooth_velocity(flags, True, amp=3.0)
    batch = {"pDiv": np.zeros_like(flags), "UDiv": U, "flags": flags, "density": synth.make_density(flags)}
    mconf = dict(dt=0.1, advectionMethod="maccormackOurs", maccormackStrength=0.6, buoyancyScale=2.0 * n / 128,
                 gravityScale=0.0, gravity=None, vorticityConfinementAmp=3.0, simMethod="jacobi", maxIter=max_iter,
                 is3D=True)
    return {k: torch.from_numpy(v) for k, v in batch.items()}, mconf


def step_rows(reps, warmup):
    from fluidnet_b200 import simulate
    from fluidnet_b200.slab import NativeSlabSimulator
    for n in (128, 256):
        for it in (34, 100):
            tb, mconf = _problem(n, it)
            sim = NativeSlabSimulator(tb, mconf, None, torch.device("cuda", 0), rank=0, world=1)
            gb = {k: v.cuda() for k, v in tb.items()}
            t_slab = _time(sim.step, reps, warmup)
            t_one = _time(lambda: simulate.simulate_fused(None, mconf, gb), reps, warmup)
            sim.close()
            print(json.dumps({"row": "step", "n": n, "maxIter": it, "slab_step_ms": round(t_slab, 4),
                              "simulate_step_ms": round(t_one, 4)}))


def block_rows(reps, warmup):
    from fluidnet_b200 import tfluids as t
    ctx = t.context()
    lib = ctx.lib

    def fields(nz, ny, nx):
        g = torch.Generator().manual_seed(3)
        flags = torch.ones(1, 1, nz, ny, nx)
        flags[torch.rand(flags.shape, generator=g) < 0.05] = 2.0
        return [x.cuda() for x in (flags, torch.randn(flags.shape, generator=g), torch.zeros(flags.shape),
                                   torch.zeros(flags.shape))]

    def block(flags, div, pa, pb, slab, z_lo, z_hi, shr, k, path):
        def run():
            if slab:
                ctx.set_slab(*slab)
            lib.tfl_jacobi_slab_block(ctx.h, t._grid(pa), t._grid(pb), t._grid(flags), t._grid(div), 1, z_lo, z_hi,
                                      shr, shr, k, path, None)
            if slab:
                ctx.clear_slab()
        return run

    # whole grids (one rank): k sweeps in one block against the single-GPU solve
    for n in (128, 256):
        flags, div, pa, pb = fields(n, n, n)
        for k in (34, 100):
            row = {"row": "block", "shape": "%d^3 whole" % n, "sweeps": k}
            for name, path in (("block_kernel", 1), ("per_sweep", 0)):
                used = C.c_int32(-1)
                ok = lib.tfl_jacobi_slab_block(ctx.h, t._grid(pa), t._grid(pb), t._grid(flags), t._grid(div), 1, 0, n,
                                               0, 0, k, path, C.byref(used)) == 0
                if ok:
                    ms = _time(block(flags, div, pa, pb, None, 0, n, 0, k, path), reps, warmup)
                    row[name + "_us_per_sweep"] = round(ms * 1000 / k, 2)
                else:
                    row[name + "_us_per_sweep"] = None
            p = torch.empty_like(div)
            ms = _time(lambda: t.solveLinearSystemJacobi(p, flags, div, True, 0, k), reps, warmup)
            row["single_gpu_solve_us_per_sweep"] = round(ms * 1000 / k, 2)
            print(json.dumps(row))
    # one interior rank's slab of 256^3 over 8 ranks (32 owned planes + 6 ghost planes per side): a block of 6 sweeps
    for nz_own, label in ((32, "256^2 x 32 owned (8 ranks)"), (64, "256^2 x 64 owned (4 ranks)")):
        halo = 6
        nz = nz_own + 2 * halo
        flags, div, pa, pb = fields(nz, 256, 256)
        slab = (100, 1000, 0, nz)
        row = {"row": "block", "shape": label, "sweeps": halo}
        for name, path in (("block_kernel", 1), ("per_sweep", 0)):
            ctx.set_slab(*slab)
            used = C.c_int32(-1)
            ok = lib.tfl_jacobi_slab_block(ctx.h, t._grid(pa), t._grid(pb), t._grid(flags), t._grid(div), 1, 1, nz - 1,
                                           1, 1, halo, path, C.byref(used)) == 0
            ctx.clear_slab()
            if ok:
                ms = _time(block(flags, div, pa, pb, slab, 1, nz - 1, 1, halo, path), reps, warmup)
                row[name + "_us_per_block"] = round(ms * 1000, 1)
            else:
                row[name + "_us_per_block"] = None
        print(json.dumps(row))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    print(json.dumps({"device": torch.cuda.get_device_name(0)}))
    block_rows(a.reps, a.warmup)
    step_rows(a.reps, a.warmup)


if __name__ == "__main__":
    main()
