"""Scene-steps per second of batched steps from graph replay, the state resident on the device (DESIGN.md section 8).

    python tests/dbg_batch_rate.py [--steps 60] [--runs 2] [--arms batched,alone] [--out FILE]

For each simMethod (convnet with the synthetic 3xTF32 model, jacobi with maxIter 34), grid (64^3 with B = 1, 2, 4,
8, 16; 128^3 with B = 1, 2, 4) and run, two arms alternate in one process:
  batched  one [B][c][z][y][x] plume-like state (geometry flags, a smooth velocity, a density and plume BCs of a
           different radius per entry), its step captured as one StepGraph and replayed;
  alone    the same B scenes as B nb = 1 states, one StepGraph each, replayed in turn.
Each arm replays --steps steps to warm up, then at least --steps steps and at least 0.3 s, timed with CUDA events; the
rate is B * steps / time.  While the timed replays run, a thread samples the SM clock (nvidia-smi clocks.sm), and each
record carries the range of those samples.
Run against another build of the library (PYTHONPATH at its tree) with `--arms batched` to time that build's batched
step.  `--profile METHOD:RES:B` instead replays each arm of that one configuration under torch.profiler (a run of its
own) and prints every kernel's device time per scene-step, largest first.  The card's name, power limit and max SM
clock are printed with the numbers."""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
if os.path.dirname(HERE) not in sys.path:
    sys.path.append(os.path.dirname(HERE))

from fluidnet_b200 import simulate, synth                            # noqa: E402
from fluidnet_b200.model import ProjectionModel                      # noqa: E402

SIZES = {64: (1, 2, 4, 8, 16), 128: (1, 2, 4)}


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:                      # pragma: no cover
        return "nvidia-smi unavailable (%s)" % e


class ClockSampler:
    """Samples the current SM clock (MHz) while `busy` is set; `take()` returns and clears the samples."""

    def __init__(self):
        self.busy = threading.Event()
        self.done = threading.Event()
        self.samples = []
        self.thread = threading.Thread(target=self._run, daemon=True)
        self.thread.start()

    def _run(self):
        while not self.done.is_set():
            if not self.busy.wait(0.05):
                continue
            try:
                v = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits", "-i", "0"],
                                   capture_output=True, text=True, timeout=30).stdout.split()[0]
            except Exception:                   # pragma: no cover
                continue
            if self.busy.is_set():              # only samples taken entirely inside a timed window count
                self.samples.append(int(v))

    def take(self):
        out, self.samples = self.samples, []
        return out

    def close(self):
        self.done.set()
        self.thread.join()


CLOCK = None


def mconf_for(method, res, model):
    m = dict(dt=0.1, advectionMethod="maccormackOurs", maccormackStrength=0.6, buoyancyScale=2.0 * res / 128,
             gravityScale=0, vorticityConfinementAmp=3.0, simMethod=method, maxIter=34, is3D=True,
             normalizeInputThreshold=float(model.threshold))
    return m


def scenes(res, n, seed=5):
    """n plume-like nb = 1 states on the host: geometry flags, a smooth velocity (|u| dt up to 0.3 cell), a density,
    plume BCs of radius 0.1 + 0.02 b."""
    out = []
    for b in range(n):
        flags = synth.make_flags(res, res, res, True, 1, geometry=True)
        U = synth.make_smooth_velocity(flags, True, amp=3.0, seed=seed + b)
        d = synth.make_density(flags, seed=seed + 100 + b)
        batch = {"pDiv": torch.zeros(flags.shape), "UDiv": torch.from_numpy(U), "flags": torch.from_numpy(flags),
                 "density": torch.from_numpy(d)}
        simulate.createPlumeBCs(batch, [1.0], 1.0 * res / 128, 0.1 + 0.02 * (b % 8))
        out.append({k: v.cpu().numpy() for k, v in batch.items() if v is not None})
    return out


def on_gpu(parts):
    return {k: torch.from_numpy(np.ascontiguousarray(np.concatenate([p[k] for p in parts]))).cuda()
            for k in parts[0]}


def timed(graphs, steps, stream, min_s=0.3):
    """(seconds, steps) of the timed replays: at least `steps` and at least `min_s` seconds."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    stream.synchronize()
    e0.record(stream)
    for _ in range(steps):                      # warm-up replays, also the estimate of one step's time
        for g in graphs:
            g.launch()
    e1.record(stream)
    e1.synchronize()
    n = max(steps, int(min_s / max(e0.elapsed_time(e1) / 1000.0 / steps, 1e-7)) + 1)
    if CLOCK is not None:
        CLOCK.busy.set()
    e0.record(stream)
    for _ in range(n):
        for g in graphs:
            g.launch()
    e1.record(stream)
    e1.synchronize()
    if CLOCK is not None:
        CLOCK.busy.clear()
    return e0.elapsed_time(e1) / 1000.0, n


def arm(name, parts, mconf, model, steps, stream):
    states = [on_gpu(parts)] if name == "batched" else [on_gpu([p]) for p in parts]
    graphs = []
    try:
        for st in states:
            simulate.simulate_fused(None, mconf, st, model)
            graphs.append(simulate.StepGraph(mconf, st, model))
        t, n = timed(graphs, steps, stream)
    finally:
        for g in graphs:
            g.close()
    return len(parts) * n / t


def profile_arm(name, parts, mconf, model, steps, stream, top=12):
    """Device time per scene-step (us) of every kernel the replays of one arm ran, largest first."""
    from collections import defaultdict
    from torch.profiler import ProfilerActivity, profile
    states = [on_gpu(parts)] if name == "batched" else [on_gpu([p]) for p in parts]
    graphs = []
    try:
        for st in states:
            simulate.simulate_fused(None, mconf, st, model)
            graphs.append(simulate.StepGraph(mconf, st, model))
        timed(graphs, 5, stream)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(steps):
                for g in graphs:
                    g.launch()
            stream.synchronize()
    finally:
        for g in graphs:
            g.close()
    per = defaultdict(float)
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            per[ev.name.replace("(anonymous namespace)::", "").split("(")[0][:90]] += ev.device_time / (steps * len(parts))
    rows = sorted(per.items(), key=lambda kv: -kv[1])
    return sum(per.values()), rows[:top]


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--steps", type=int, default=60)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--methods", default="convnet,jacobi")
    ap.add_argument("--arms", default="batched,alone")
    ap.add_argument("--tag", default="", help="a label for this build in the JSON lines")
    ap.add_argument("--out")
    ap.add_argument("--profile", metavar="METHOD:RES:B", help="profile the arms of one configuration instead")
    args = ap.parse_args(argv)
    global CLOCK
    torch.cuda.set_device(0)
    print("card (max SM clock): %s" % card())
    model = ProjectionModel(synth.make_model(True)["layers"], True)
    model.set_mode("tf32x3")
    stream = torch.cuda.Stream()
    if args.profile:
        method, res, B = args.profile.split(":")
        res, B = int(res), int(B)
        mconf = mconf_for(method, res, model)
        pool = scenes(res, B)
        with torch.cuda.stream(stream):
            for a in args.arms.split(","):
                total, rows = profile_arm(a, pool, mconf, model if method == "convnet" else None, args.steps, stream)
                print("%s %s %s: %.1f us of kernels per scene-step" % (args.tag, args.profile, a, total))
                for name, us in rows:
                    print("  %9.2f  %s" % (us, name))
        return
    recs = []
    CLOCK = ClockSampler()
    try:
        run_table(args, model, stream, recs)
    finally:
        CLOCK.close()
    if args.out:
        with open(args.out, "a") as f:
            f.write(json.dumps({"card": card(), "records": recs}) + "\n")


def run_table(args, model, stream, recs):
    with torch.cuda.stream(stream):
        for method in args.methods.split(","):
            for res, bs in SIZES.items():
                mconf = mconf_for(method, res, model)
                pool = scenes(res, max(bs))
                for B in bs:
                    rates = {a: [] for a in args.arms.split(",")}
                    for _ in range(args.runs):
                        for a in rates:
                            rates[a].append(arm(a, pool[:B], mconf, model if method == "convnet" else None,
                                                args.steps, stream))
                    clk = CLOCK.take()
                    rec = {"tag": args.tag, "method": method, "res": res, "B": B,
                           "scene_steps_per_s": {a: [round(r, 1) for r in v] for a, v in rates.items()},
                           "sm_clock_mhz": [min(clk), max(clk), len(clk)] if clk else None}
                    recs.append(rec)
                    print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
