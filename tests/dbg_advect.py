"""Kernel-tuning script (not a test): the two advection operators alone on the bench state after a few
steps, timed with CUDA events.  Run under ncu for the source-level counters:
  ncu --set full --import-source on -k regex:k_advect -c 8 -o gpurun_out/advect python tests/dbg_advect.py 128 1
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from fluidnet_b200 import tfluids, simulate, model as fmodel  # noqa: E402

n = int(sys.argv[1]) if len(sys.argv) > 1 else 128
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 20
velocity = sys.argv[3] if len(sys.argv) > 3 else "smooth"
batch_np, mconf, mnp = bench.make_problem(n, velocity)
gb = {k: torch.from_numpy(v.copy()).cuda() for k, v in batch_np.items()}
gm = fmodel.ProjectionModel(mnp["layers"], True)
for _ in range(8):
    simulate.simulate_fused(None, mconf, gb, gm)
torch.cuda.synchronize()
U, fl, rho = gb["UDiv"], gb["flags"], gb["density"]
print("max|U| dt = %.3f cells" % (float(U.abs().max()) * mconf["dt"]), flush=True)
Ud, rd = torch.empty_like(U), torch.empty_like(rho)
flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device="cuda")


def timed(fn):
    for _ in range(2):
        fn()
    ts = []
    for _ in range(reps):
        flush.fill_(0.0)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts)) * 1e3


import ctypes as C
ctx = tfluids.context()
ctx.lib.tfl_debug_advect_tile.argtypes = [C.c_void_p, C.c_int]
ref = None
for mode in (0, 1, 2):
    if len(sys.argv) > 4 and mode != int(sys.argv[4]):
        continue
    ctx.lib.tfl_debug_advect_tile(ctx.h, mode)
    t = timed(lambda: tfluids.advectVel(0.1, U, fl, "maccormackOurs", Ud, 0.6))
    if ref is None:
        ref = Ud.clone()
    same = torch.equal(ref.view(torch.int32), Ud.view(torch.int32))
    print("advectVel mode %d: %.1f us  %s" % (mode, t, "== first" if same else "DIFFERS"), flush=True)
ctx.lib.tfl_debug_advect_tile(ctx.h, -1)
ref = None
for mode in (0, 1, 2):
    ctx.lib.tfl_debug_advect_tile(ctx.h, mode)
    t = timed(lambda: tfluids.advectScalar(0.1, rho, U, fl, "maccormackOurs", rd, False, 0.6))
    if ref is None:
        ref = rd.clone()
    same = torch.equal(ref.view(torch.int32), rd.view(torch.int32))
    print("advectScalar mode %d: %.1f us  %s" % (mode, t, "== first" if same else "DIFFERS"), flush=True)
ctx.lib.tfl_debug_advect_tile(ctx.h, -1)
t_v = timed(lambda: tfluids.advectVel(0.1, U, fl, "maccormackOurs", Ud, 0.6))
t_s = timed(lambda: tfluids.advectScalar(0.1, rho, U, fl, "maccormackOurs", rd, False, 0.6))
print("advectVel %.1f us   advectScalar %.1f us   (%d^3, %s velocity, L2 flushed)" % (t_v, t_s, n, velocity), flush=True)
assert tfluids.context().trace_faults() == 0
