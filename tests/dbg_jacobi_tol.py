"""Timing script (not a test): converged Jacobi solves (pTol 1e-5, maxIter 100000, the reference's acceptance test,
tfluids/test_tfluids.lua:907-963) on the plume's divergence at 64^3, 128^3 and 256^3, through the direct call
(tfl_solve_linear_system_jacobi, one wait at the end), the _dev call (ended by a stream synchronise) and a replayed
CUDA graph of the _dev call.  With --parent-lib, a libtfl.so built from an earlier commit runs the same solves through
its own direct call (the per-sweep host loop there), alternated with the others in every round; p must then agree bit
for bit.  Prints the GPU's name, power limit and clocks beside the numbers, and one JSON line.

    python tests/dbg_jacobi_tol.py [--sizes 64,128,256] [--rounds 5] [--parent-lib /path/to/libtfl.so]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from fluidnet_b200 import tfluids                      # noqa: E402
from fluidnet_b200._lib import Grid                    # noqa: E402
from scenes import plume_batch                         # noqa: E402

TOL, MAX_ITER = 1e-5, 100000


def gpu_info():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[torch.cuda.current_device()] if r.returncode == 0 else "unknown"


class ParentLib:
    """The direct call of a libtfl.so from an earlier commit, on its own context and on torch's current stream."""

    def __init__(self, path):
        self.lib = C.CDLL(path)
        self.lib.tfl_create.argtypes = [C.POINTER(C.c_void_p), C.c_int]
        self.lib.tfl_set_stream.argtypes = [C.c_void_p, C.c_void_p]
        self.lib.tfl_last_error.argtypes = [C.c_void_p]
        self.lib.tfl_last_error.restype = C.c_char_p
        G = C.POINTER(Grid)
        self.lib.tfl_solve_linear_system_jacobi.argtypes = [C.c_void_p, G, G, G, C.c_int, C.c_float, C.c_int,
                                                            C.POINTER(C.c_float), C.POINTER(C.c_int)]
        self.h = C.c_void_p()
        assert self.lib.tfl_create(C.byref(self.h), torch.cuda.current_device()) == 0

    def solve(self, p, f, d):
        s = torch.cuda.current_stream().cuda_stream
        assert self.lib.tfl_set_stream(self.h, C.c_void_p(s if s else 1)) == 0
        res, it = C.c_float(0), C.c_int(0)
        rc = self.lib.tfl_solve_linear_system_jacobi(self.h, C.byref(tfluids._grid(p)), C.byref(tfluids._grid(f)),
                                                     C.byref(tfluids._grid(d)), 1, TOL, MAX_ITER, C.byref(res),
                                                     C.byref(it))
        assert rc == 0, self.lib.tfl_last_error(self.h)
        return res.value, it.value


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="64,128,256")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--parent-lib", default=None)
    a = ap.parse_args()
    info = gpu_info()
    print("GPU:", info)
    parent = ParentLib(a.parent_lib) if a.parent_lib else None
    stream = torch.cuda.Stream()            # a non-default stream, so that the _dev call can be captured
    results = {}
    with torch.cuda.stream(stream):
        for n in (int(s) for s in a.sizes.split(",")):
            batch = plume_batch(n)
            f = torch.from_numpy(batch["flags"]).cuda()
            U = torch.from_numpy(batch["UDiv"]).cuda()
            d = torch.zeros_like(f)
            tfluids.velocityDivergenceForward(U, f, d)
            p_direct, p_dev, p_graph, p_parent = (torch.zeros_like(f) for _ in range(4))
            direct = lambda: (tfluids.solveLinearSystemJacobi(p_direct, f, d, True, TOL, MAX_ITER),
                              tfluids.solveLinearSystemJacobi.last_iterations)
            device = lambda: tfluids.solveLinearSystemJacobiDevice(p_dev, f, d, True, TOL, MAX_ITER)
            device()
            graph = torch.cuda.CUDAGraph()
            torch.cuda.synchronize()
            with torch.cuda.graph(graph, stream=stream):
                g_res, g_it = tfluids.solveLinearSystemJacobiDevice(p_graph, f, d, True, TOL, MAX_ITER)
            runs = {"direct": direct, "dev": device, "graph": graph.replay}
            if parent:
                runs["parent"] = lambda: parent.solve(p_parent, f, d)
            times = {k: [] for k in runs}
            outs = {}
            for _ in range(a.rounds + 1):        # the first round warms up
                for k, fn in runs.items():
                    t, outs[k] = timed(fn)
                    times[k].append(t)
            res, it = outs["direct"]
            dev_res, dev_it = outs["dev"]
            same = {"dev": torch.equal(p_dev, p_direct) and float(dev_res.item()) == res and int(dev_it.item()) == it,
                    "graph": torch.equal(p_graph, p_direct) and float(g_res.item()) == res and int(g_it.item()) == it}
            if parent:
                pres, pit = outs["parent"]
                same["parent"] = torch.equal(p_parent, p_direct) and pit == it and abs(pres - res) <= 1e-6 * abs(res)
            med = {k: float(np.median(v[1:])) * 1e3 for k, v in times.items()}
            spread = {k: (float(np.min(v[1:])) * 1e3, float(np.max(v[1:])) * 1e3) for k, v in times.items()}
            results[n] = dict(iterations=it, residual=res, ms=med, ms_range=spread, same_as_direct=same,
                              us_per_sweep={k: v * 1e3 / max(it, 1) for k, v in med.items()})
            print("%d^3: %d sweeps, residual %.3g" % (n, it, res))
            for k in runs:
                print("  %-7s %9.2f ms  (%.2f .. %.2f)  %.2f us/sweep" % (k, med[k], spread[k][0], spread[k][1],
                                                                         results[n]["us_per_sweep"][k]))
            print("  bit-identical to the direct call:", same)
    print(json.dumps({"gpu": info, "tol": TOL, "max_iter": MAX_ITER, "rounds": a.rounds, "sizes": results}))


if __name__ == "__main__":
    main()
