"""What the step monitor costs on the replayed plume step (DESIGN.md section 6b).

    python tests/dbg_monitor_rate.py [--sizes 128 256] [--runs 3] [--out FILE]

For each size: the plume step with the synthetic convnet model, captured once as a step graph and replayed, in three
arms that alternate run by run -- no monitor, the monitor recording every frame (records drained without waiting),
and the synchronous alternative (velocityDivergenceForward into a spare field and a torch norm every frame) -- and
the monitor's two kernels alone, timed with CUDA events after an L2 flush, against the 16 B/cell HBM bound (U 12 +
flags 4 bytes per cell at 3.35 TB/s), and each of the two kernels' share of that time from a separate run under
torch.profiler (device time per kernel name, same L2 flush).  The card's name, power limit and max SM clock are
printed with the numbers."""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from fluidnet_b200 import monitor, scene, simulate, synth, tfluids   # noqa: E402
from fluidnet_b200.model import ProjectionModel                      # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:                      # pragma: no cover
        out = "nvidia-smi unavailable (%s)" % e
    return out


def plume(res, model):
    mconf = scene.scene_mconf(res, "convnet")
    mconf["normalizeInputThreshold"] = float(model.threshold)
    zeros = lambda c: torch.zeros(1, c, res, res, res, dtype=torch.float32, device="cuda")   # noqa: E731
    batch = {"pDiv": zeros(1), "UDiv": zeros(3), "flags": torch.from_numpy(scene.scene_flags(res)).cuda(),
             "density": zeros(1)}
    simulate.createPlumeBCs(batch, scene.DENSITY_VAL, 1.0 * (res / 128), scene.PLUME_RAD)
    return mconf, batch


def run_arm(arm, graph, batch, mon, div, steps, stream):
    stream.synchronize()
    t0 = time.perf_counter()
    norms = []
    for _ in range(steps):
        graph.launch()
        if arm == "monitor":
            mon.record(batch)
            mon.drain()
        elif arm == "sync":
            tfluids.velocityDivergenceForward(batch["UDiv"], batch["flags"], div)
            norms.append(div.norm().item())
    if arm == "monitor":
        mon.drain(wait=True)
    stream.synchronize()
    return (time.perf_counter() - t0) / steps


def kernel_time(mon, batch, reps, stream):
    flush = torch.empty(64 << 20, dtype=torch.float32, device="cuda")     # 256 MB, past the 50 MB L2
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    for e0, e1 in ev:
        flush.fill_(1.0)
        e0.record(stream)
        mon.record(batch)
        e1.record(stream)
        mon.take(wait=True)
    stream.synchronize()
    ts = sorted(e0.elapsed_time(e1) * 1e3 for e0, e1 in ev)
    return ts[len(ts) // 2], ts[0]


def kernel_split(mon, batch, reps, stream):
    """Median device time (us) of k_monitor_chunks and k_monitor_finish, from a torch.profiler run of its own."""
    from torch.profiler import ProfilerActivity, profile
    flush = torch.empty(64 << 20, dtype=torch.float32, device="cuda")
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            flush.fill_(1.0)
            mon.record(batch)
            mon.take(wait=True)
        stream.synchronize()
    times = {"k_monitor_chunks": [], "k_monitor_finish": []}
    for e in prof.events():
        for k in times:
            if k in e.name and e.device_type.name == "CUDA":
                times[k].append(e.time_range.elapsed_us())
    return {k: (sorted(v)[len(v) // 2] if v else None) for k, v in times.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[128, 256])
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out")
    args = ap.parse_args()
    lines = ["card: " + card()]
    print(lines[0], flush=True)
    model = ProjectionModel(synth.make_model(True)["layers"], True)
    stream = torch.cuda.Stream()
    results = []
    with torch.cuda.stream(stream):
        for res in args.sizes:
            steps = {128: 60}.get(res, 20)
            mconf, batch = plume(res, model)
            simulate.simulate_fused(None, mconf, batch, model)
            graph = simulate.StepGraph(mconf, batch, model)
            mon = monitor.StepMonitor(None, batch, capacity=steps + 1)
            div = torch.empty_like(batch["pDiv"])
            for arm in ("none", "monitor", "sync"):            # warm-up of every arm
                run_arm(arm, graph, batch, mon, div, 3, stream)
            per = {"none": [], "monitor": [], "sync": []}
            for _ in range(args.runs):
                for arm in per:
                    per[arm].append(run_arm(arm, graph, batch, mon, div, steps, stream) * 1e3)
            med, best = kernel_time(mon, batch, 50, stream)
            split = kernel_split(mon, batch, 20, stream)
            bound = res ** 3 * 16 / HBM_BYTES_PER_S * 1e6
            r = {"res": res, "steps_per_run": steps, "ms_per_step": per,
                 "monitor_cost_pct": 100.0 * (min(per["monitor"]) - min(per["none"])) / min(per["none"]),
                 "sync_cost_pct": 100.0 * (min(per["sync"]) - min(per["none"])) / min(per["none"]),
                 "record_kernels_us_median": med, "record_kernels_us_best": best, "hbm_bound_us": bound,
                 "share_of_bound_median": bound / med, "profiler_kernel_us_median": split}
            results.append(r)
            lines.append(json.dumps(r))
            print(lines[-1], flush=True)
            mon.close()
            graph.close()
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
