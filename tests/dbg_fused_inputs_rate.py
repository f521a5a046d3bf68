"""Step time with each input block of the projection network (3xTF32): the fused step replayed from a step graph
against the operator sequence (simulate.simulate, enqueued from Python), at 64^3 and 128^3, the two alternated in
one process, CUDA events around `iters` steps, best of `reps` alternations.  The SM clock is sampled (nvidia-smi,
every 100 ms) while the timed steps run, and the card's name and power limit are printed with the numbers.
Usage: python tests/dbg_fused_inputs_rate.py [iters] [reps]"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import oracle  # noqa: E402
from fluidnet_b200 import model as fmodel, simulate, synth  # noqa: E402

iters = int(sys.argv[1]) if len(sys.argv) > 1 else 50
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
BLOCKS = {
    "default": {},
    "pDiv+UDiv+div": {"inputChannels": {"UDiv": True}},
    "UDiv": {"inputChannels": {"pDiv": False, "UDiv": True, "div": False}},
    "norm": {"normalizeInputFunc": "norm"},
    "chan-pDiv": {"normalizeInputChan": "pDiv"},
    "chan-div": {"normalizeInputChan": "div"},
    "skip": {"addPressureSkip": True},
    "no-normalize": {"normalizeInput": False},
}


def smi(query):
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=" + query, "--format=csv,noheader", "-i",
                               str(torch.cuda.current_device())], capture_output=True, text=True,
                              timeout=30).stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


class ClockSampler:
    """SM clock (MHz) every 100 ms while the block runs."""

    def __enter__(self):
        try:
            self.p = subprocess.Popen(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits",
                                       "-lms", "100", "-i", str(torch.cuda.current_device())],
                                      stdout=subprocess.PIPE, text=True)
        except OSError:
            self.p = None
        self.mhz = []
        return self

    def __exit__(self, *exc):
        if self.p is not None:
            self.p.terminate()
            out, _ = self.p.communicate(timeout=30)
            self.mhz = [int(x) for x in out.split() if x.isdigit()]


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def state(n):
    flags = synth.make_flags(n, n, n, True, nb=1, geometry=True)
    U = synth.make_smooth_velocity(flags, True, amp=2.0)
    oracle.Oracle().setWallBcsForward(U, flags)
    base = {"pDiv": ((np.random.RandomState(3).rand(*flags.shape) - 0.5) * 0.2).astype(np.float32), "UDiv": U,
            "flags": flags, "density": synth.make_density(flags)}
    oracle.create_plume_bcs(base, [1.0], n / 128.0 * 4, 0.15)
    return base


def main():
    name, limit = torch.cuda.get_device_name(), smi("power.limit")
    print("card: %s, power limit %s; %d steps per window, best of %d" % (name, limit, iters, reps), flush=True)
    out = {"card": name, "power_limit": limit, "ms": {}}
    for n in (64, 128):
        mconf = oracle.default_mconf(dt=0.1, maccormackStrength=0.6, buoyancyScale=2.0 * n / 128,
                                     vorticityConfinementAmp=3.0, simMethod="convnet")
        base = state(n)
        for block, kw in BLOCKS.items():
            gm = fmodel.ProjectionModel.from_model(synth.make_model(True, inputs=dict(kw) if kw else None))
            stream = torch.cuda.Stream()
            torch.cuda.synchronize()
            with torch.cuda.stream(stream):
                fused = {k: torch.from_numpy(v.copy()).cuda() for k, v in base.items()}
                ops = {k: torch.from_numpy(v.copy()).cuda() for k, v in base.items()}
                # the operator sequence's projection scratch is the larger one: grow the arena before the capture
                simulate.simulate(None, mconf, ops, gm)
                simulate.simulate_fused(None, mconf, fused, gm)
                graph = simulate.StepGraph(mconf, fused, gm)
                for _ in range(3):
                    graph.launch()
                    simulate.simulate(None, mconf, ops, gm)
                stream.synchronize()
                best = {"fused graph": float("inf"), "operators": float("inf")}
                with ClockSampler() as clk:
                    for _ in range(reps):
                        best["fused graph"] = min(best["fused graph"], timed(graph.launch))
                        best["operators"] = min(best["operators"], timed(lambda: simulate.simulate(None, mconf, ops, gm)))
                graph.close()
            mhz = "%d-%d MHz" % (min(clk.mhz), max(clk.mhz)) if clk.mhz else "not sampled"
            out["ms"]["%d/%s" % (n, block)] = {k: round(v, 4) for k, v in best.items()}
            print("%3d^3 %-14s fused graph %7.3f ms   operators %7.3f ms   SM clock %s" % (
                n, block, best["fused graph"], best["operators"], mhz), flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
