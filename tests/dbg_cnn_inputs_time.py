"""Cost of the projection network's input-block options on the GPU (CUDA events, steady state):
  * tfl_cnn_project at n^3 in modes fp32 / tf32 / tf32x3 with the default block {pDiv, div, flags}, with
    {pDiv, UDiv, div, flags} (two-plane tensor-core input, 6-channel fp32 layer 1) and with the default block plus
    addPressureSkip (one more pass over p_net);
  * one tfl_simulate_step with the {pDiv, UDiv, div, flags} model (per-operator step) against the default model's
    fused step.
Prints the card's name and power limit with the numbers.  Usage: python tests/dbg_cnn_inputs_time.py [n] [iters]"""
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import oracle  # noqa: E402
from fluidnet_b200 import model as fmodel, simulate, synth  # noqa: E402

n = int(sys.argv[1]) if len(sys.argv) > 1 else 128
iters = int(sys.argv[2]) if len(sys.argv) > 2 else 20
ALL = dict(pDiv=True, UDiv=True, div=True, flags=True)
BLOCKS = {"default": {}, "pDiv+UDiv+div": dict(inputChannels=ALL), "default+skip": dict(addPressureSkip=True)}


def card():
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                                str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
    except (OSError, subprocess.SubprocessError):
        limit = "unknown"
    return torch.cuda.get_device_name(), limit.strip() or "unknown"


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


def main():
    name, limit = card()
    print("card: %s, power limit %s; n = %d, %d iterations per number" % (name, limit, n, iters), flush=True)
    flags_np = synth.make_flags(n, n, n, True, nb=1, geometry=True)
    U_np = synth.make_smooth_velocity(flags_np, True, amp=2.0)
    flags, U = torch.from_numpy(flags_np).cuda(), torch.from_numpy(U_np).cuda()
    p = torch.zeros_like(flags)
    out = {"card": name, "power_limit": limit, "n": n, "project_ms": {}, "step_ms": {}}
    for block, kw in BLOCKS.items():
        mnp = synth.make_model(True, inputs=dict(kw) if kw else None)
        gm = fmodel.ProjectionModel(mnp["layers"], True, **kw)
        po, Uo = torch.empty_like(p), torch.empty_like(U)
        for mode in ("fp32", "tf32", "tf32x3"):
            gm.set_mode(mode)
            ms = timed(lambda: gm.forward((p, U, flags), out=(po, Uo)))
            out["project_ms"]["%s/%s" % (block, mode)] = round(ms, 4)
            print("tfl_cnn_project %-14s %-7s %8.3f ms" % (block, mode, ms), flush=True)
    mconf = oracle.default_mconf(dt=0.1, maccormackStrength=0.6, buoyancyScale=2.0 * n / 128,
                                 vorticityConfinementAmp=3.0, simMethod="convnet")
    base = {"pDiv": flags_np * 0, "UDiv": U_np, "flags": flags_np, "density": synth.make_density(flags_np)}
    oracle.create_plume_bcs(base, [1.0], n / 128.0 * 4, 0.15)
    for block in ("default", "pDiv+UDiv+div"):
        kw = BLOCKS[block]
        mnp = synth.make_model(True, inputs=dict(kw) if kw else None)
        gm = fmodel.ProjectionModel(mnp["layers"], True, **kw)
        batch = {k: torch.from_numpy(v.copy()).cuda() for k, v in base.items()}
        ms = timed(lambda: simulate.simulate_fused(None, mconf, batch, gm))
        out["step_ms"][block] = round(ms, 4)
        print("tfl_simulate_step %-14s (tf32x3) %8.3f ms" % (block, ms), flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
