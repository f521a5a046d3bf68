"""Cost of batch normalization in the projection network on the GPU (CUDA events, steady state), on the 3-D 'default'
graph at n^3:
  * tfl_cnn_project in fp32 / tf32 / tf32x3 without BN, with running statistics and with batch statistics;
  * one tfl_simulate_step with each in fp32 (per-operator step) and tf32x3 (fused step).
Prints the card's name and power limit with the numbers.  Usage: python tests/dbg_bn_time.py [n] [iters]"""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import oracle  # noqa: E402
from dbg_cnn_inputs_time import card  # noqa: E402
from fluidnet_b200 import model as fmodel, simulate, synth  # noqa: E402

n = int(sys.argv[1]) if len(sys.argv) > 1 else 128
iters = int(sys.argv[2]) if len(sys.argv) > 2 else 20


def timed(fn, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def models():
    """(name, model, modes) of the three variants."""
    plain = synth.make_model(True)
    yield "no BN", fmodel.ProjectionModel(plain["layers"], True), ("fp32", "tf32", "tf32x3")
    for name, train in (("BN running", False), ("BN batch", True)):
        m = synth.make_model(True, batch_norm={"train": train})
        yield name, fmodel.ProjectionModel(m["layers"], True, batchNorm=m["batchNorm"]), ("fp32", "tf32", "tf32x3")


def main():
    name, limit = card()
    print("card: %s, power limit %s; n = %d, %d iterations per number" % (name, limit, n, iters), flush=True)
    flags_np = synth.make_flags(n, n, n, True, nb=1, geometry=True)
    U_np = synth.make_smooth_velocity(flags_np, True, amp=2.0)
    flags, U = torch.from_numpy(flags_np).cuda(), torch.from_numpy(U_np).cuda()
    p = torch.zeros_like(flags)
    out = {"card": name, "power_limit": limit, "n": n, "project_ms": {}, "step_ms": {}}
    mconf = oracle.default_mconf(dt=0.1, maccormackStrength=0.6, buoyancyScale=2.0 * n / 128,
                                 vorticityConfinementAmp=3.0, simMethod="convnet")
    base = {"pDiv": flags_np * 0, "UDiv": U_np, "flags": flags_np, "density": synth.make_density(flags_np)}
    oracle.create_plume_bcs(base, [1.0], n / 128.0 * 4, 0.15)
    for label, gm, modes in models():
        po, Uo = torch.empty_like(p), torch.empty_like(U)
        for mode in modes:
            gm.set_mode(mode)
            ms = timed(lambda: gm.forward((p, U, flags), out=(po, Uo)))
            out["project_ms"]["%s/%s" % (label, mode)] = round(ms, 4)
            print("tfl_cnn_project   %-11s %-7s %8.3f ms" % (label, mode, ms), flush=True)
            if mode in ("fp32", "tf32x3"):
                batch = {k: torch.from_numpy(v.copy()).cuda() for k, v in base.items()}
                ms = timed(lambda: simulate.simulate_fused(None, mconf, batch, gm))
                out["step_ms"]["%s/%s" % (label, mode)] = round(ms, 4)
                print("tfl_simulate_step %-11s %-7s %8.3f ms" % (label, mode, ms), flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
