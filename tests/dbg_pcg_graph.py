"""The PCG step launched directly (tfl_simulate_step, which waits for the host every fourth iteration) against the same
step replayed from a step graph (the iteration loop a conditional node on the device).

    python tests/dbg_pcg_graph.py [--steps 40] [--reps 3] [--out results.json]

The plume of the demo scene (scene.scene_mconf: buoyancy, vorticity confinement, maccormackOurs) on the synthetic
geometry at 64^3 and 128^3, maxIter 34 (the scene's) and 100 (the reference's default).  For each, the two arms run
alternately `reps` times from the same state, `steps` steps each, and print
  - device ms per step: CUDA events around the steps on the step stream;
  - host busy ms per step: the host clock from the first call until the last call returns (before the final
    synchronise): how long the host is held by enqueueing the steps;
  - the longest iteration count of the last step's solve (pcg_status for the replay);
and the card's name and power limit.  Both arms must leave the same bits."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from fluidnet_b200 import scene, simulate, synth          # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown (%s)" % q.stderr.strip()


def problem(n, max_iter):
    flags = synth.make_flags(n, n, n, True, nb=1, geometry=True)
    batch = {"pDiv": np.zeros_like(flags), "UDiv": synth.make_smooth_velocity(flags, True, amp=2.0), "flags": flags,
             "density": synth.make_density(flags)}
    gb = {k: torch.from_numpy(v.copy()).cuda() for k, v in batch.items()}
    simulate.createPlumeBCs(gb, [1.0], n / 128.0, 0.15)
    mconf = scene.scene_mconf(n, "pcg")
    mconf["maxIter"] = max_iter
    return gb, mconf


def run_arm(arm, graph, gb, mconf, start, steps, stream):
    for k, v in start.items():
        gb[k].copy_(v)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    stream.synchronize()
    t0 = time.perf_counter()
    e0.record(stream)
    for _ in range(steps):
        if arm == "replay":
            graph.launch()
        else:
            simulate.simulate_fused(None, mconf, gb)
    e1.record(stream)
    busy = time.perf_counter() - t0
    stream.synchronize()
    it = graph.pcg_status()[1] if arm == "replay" else None
    return e0.elapsed_time(e1) / steps, 1000.0 * busy / steps, it


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out")
    args = ap.parse_args()
    torch.cuda.init()
    out = {"card": card(), "steps": args.steps, "runs": []}
    print("card:", out["card"])
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        for n in (64, 128):
            for max_iter in (34, 100):
                gb, mconf = problem(n, max_iter)
                for _ in range(3):                       # warm up, and move the plume off its initial state
                    simulate.simulate_fused(None, mconf, gb)
                graph = simulate.StepGraph(mconf, gb)
                start = {k: v.clone() for k, v in gb.items() if v is not None}
                ends = {}
                res = {"direct": [], "replay": []}
                for _ in range(args.reps):
                    for arm in ("direct", "replay"):
                        ms, busy, it = run_arm(arm, graph, gb, mconf, start, args.steps, stream)
                        res[arm].append((ms, busy))
                        ends[arm] = {k: gb[k].clone() for k in ("pDiv", "UDiv", "density")}
                        if it is not None:
                            res["iterations"] = it
                graph.close()
                same = all(torch.equal(ends["direct"][k].view(torch.int32), ends["replay"][k].view(torch.int32))
                           for k in ends["direct"])
                row = {"n": n, "maxIter": max_iter, "bits_equal": same, "iterations_last_step": res.get("iterations")}
                for arm in ("direct", "replay"):
                    row[arm + "_ms"] = [round(a, 3) for a, _ in res[arm]]
                    row[arm + "_host_busy_ms"] = [round(b, 3) for _, b in res[arm]]
                out["runs"].append(row)
                print(json.dumps(row))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
