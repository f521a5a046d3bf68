"""What replaying the z-slab step from a CUDA graph saves on one rank (DESIGN.md section 5).

    python tests/dbg_slab_graph_rate.py [--sizes 64 128 256] [--methods convnet jacobi] [--runs 3] [--out FILE]

For each size and simMethod: the demo's plume (scene.scene_mconf: maxIter 34 for 'jacobi', the synthetic 3xTF32 model
for 'convnet') on a world-1 NativeSlabSimulator, stepped directly (tfl_slab_sim_step) and replayed (SlabStepGraph) in
windows that alternate run by run.  Per window: device ms/step from CUDA events around the window, and host ms/step
around the enqueue alone (the loop of step() / launch() calls, before the synchronise).  The card's name, power limit
and SM clocks are read in the same call.  Ranks that share one GPU time-slice it, so multi-rank rates are not measured
here."""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from fluidnet_b200 import scene, simulate, synth                 # noqa: E402
from fluidnet_b200.model import ProjectionModel                   # noqa: E402
from fluidnet_b200.slab import NativeSlabSimulator, SlabStepGraph  # noqa: E402


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:                      # pragma: no cover
        out = "nvidia-smi unavailable (%s)" % e
    return out


def plume_sim(res, method, model):
    mconf = scene.scene_mconf(res, method)
    if model is not None:
        mconf["normalizeInputThreshold"] = float(model.threshold)
    zeros = lambda c: torch.zeros(1, c, res, res, res, dtype=torch.float32)    # noqa: E731
    batch = {"pDiv": zeros(1), "UDiv": zeros(3), "flags": torch.from_numpy(scene.scene_flags(res)), "density": zeros(1)}
    simulate.createPlumeBCs(batch, scene.DENSITY_VAL, 1.0 * (res / 128), scene.PLUME_RAD)
    return NativeSlabSimulator(batch, mconf, None, torch.device("cuda", 0), 0, 1, scene.SLAB_MARGIN,
                               model=model if method == "convnet" else None)


def window(run, steps, stream):
    """(device ms/step, host ms/step around the enqueue) of `steps` calls of run()."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    stream.synchronize()
    e0.record(stream)
    t0 = time.perf_counter()
    for _ in range(steps):
        run()
    t1 = time.perf_counter()
    e1.record(stream)
    stream.synchronize()
    return e0.elapsed_time(e1) / steps, 1e3 * (t1 - t0) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[64, 128, 256])
    ap.add_argument("--methods", nargs="+", default=["convnet", "jacobi"])
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out")
    args = ap.parse_args()
    lines = ["card (name, power limit, SM clock, max SM clock): " + card()]
    print(lines[0], flush=True)
    model = ProjectionModel(synth.make_model(True)["layers"], True)
    model.set_mode("tf32x3")
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        for method in args.methods:
            for res in args.sizes:
                steps = {64: 100, 128: 40}.get(res, 12)
                sim = plume_sim(res, method, model)
                sim.step()
                graph = SlabStepGraph(sim)
                arms = {"direct": sim.step, "replay": graph.launch}
                for run in arms.values():                     # warm-up of both arms
                    window(run, 3, stream)
                per = {k: [] for k in arms}
                for _ in range(args.runs):
                    for k, run in arms.items():
                        per[k].append(window(run, steps, stream))
                sim.check()
                best = {k: (min(d for d, _ in v), min(h for _, h in v)) for k, v in per.items()}
                r = {"method": method, "res": res, "steps_per_window": steps,
                     "device_ms_per_step": {k: [round(d, 4) for d, _ in v] for k, v in per.items()},
                     "host_enqueue_ms_per_step": {k: [round(h, 4) for _, h in v] for k, v in per.items()},
                     "best_device_ms": {k: round(b[0], 4) for k, b in best.items()},
                     "best_host_ms": {k: round(b[1], 4) for k, b in best.items()}}
                lines.append(json.dumps(r))
                print(lines[-1], flush=True)
                graph.close()
                sim.close()
    lines.append("card after the runs: " + card())
    print(lines[-1], flush=True)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
