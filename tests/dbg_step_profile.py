"""Per-kernel profile of the bench.py headline step: make_problem(128) replayed from a CUDA graph
(simulate.StepGraph), L2 flushed between steps as bench.py does, under torch.profiler with CUDA
activities.  Prints the card, its power limit and SM clocks, then one row per kernel: calls per step,
mean us per call, us per step and share of the summed kernel time of a step.

    python tests/dbg_step_profile.py [--grid 128] [--steps 50] [--json OUT.json]"""
import argparse
import json
import os
import subprocess
import sys
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=10).stdout.strip()
    return dict(zip(q.split(","), [x.strip() for x in out.split(",")]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--grid", type=int, default=128)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--json", default=None, help="also write the table as JSON here")
    args = ap.parse_args()

    import torch
    from torch.profiler import profile, ProfilerActivity
    import bench
    from fluidnet_b200 import simulate, model as fmodel

    assert torch.cuda.is_available(), "the profile needs a CUDA device"
    torch.cuda.set_device(0)
    batch_np, mconf, mnp = bench.make_problem(args.grid)
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        gb = {k: torch.from_numpy(v.copy()).cuda() for k, v in batch_np.items()}
        gm = fmodel.ProjectionModel(mnp["layers"], True)
        flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device="cuda")
        for _ in range(3):
            simulate.simulate_fused(None, mconf, gb, gm)
        graph = simulate.StepGraph(mconf, gb, gm)
        for _ in range(5):
            graph.launch()
        stream.synchronize()
        info = card()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.steps):
                flush.fill_(0.0)
                graph.launch()
            stream.synchronize()
        info_after = card()
        graph.close()

    tot = defaultdict(float)
    cnt = defaultdict(int)
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        name = ev.name
        if "fill" in name.lower() or name.startswith("Memset") or name.startswith("Memcpy"):
            continue                                    # the L2 flush between steps is not part of the step
        tot[name] += ev.device_time
        cnt[name] += 1
    assert tot, "the profiler recorded no kernels of the step"
    step_us = sum(tot.values()) / args.steps
    rows = sorted(tot, key=lambda k: -tot[k])
    print("card: %s, power limit %s, SM clock %s (max %s) before / %s after the profiled steps"
          % (info.get("name"), info.get("power.limit"), info.get("clocks.sm"), info.get("clocks.max.sm"),
             info_after.get("clocks.sm")))
    print("grid %d^3, %d graph replays, summed kernel time %.1f us per step" % (args.grid, args.steps, step_us))
    print("%-60s %7s %9s %9s %6s" % ("kernel", "calls", "us/call", "us/step", "share"))
    table = []
    for k in rows:
        short = k if len(k) <= 60 else k[:57] + "..."
        per_step = tot[k] / args.steps
        r = {"kernel": k, "calls_per_step": cnt[k] / args.steps, "us_per_call": tot[k] / cnt[k],
             "us_per_step": per_step, "share": per_step / step_us}
        table.append(r)
        print("%-60s %7.2f %9.1f %9.1f %5.1f%%" % (short, r["calls_per_step"], r["us_per_call"], per_step,
                                                  100 * r["share"]))
    conv = sum(r["us_per_step"] for r in table if "k_conv3_tc" in r["kernel"])
    print("k_conv3_tc total: %.1f us per step (%.1f%%)" % (conv, 100 * conv / step_us))
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump({"card": info, "card_after": info_after, "grid": args.grid, "steps": args.steps,
                       "step_kernel_us": step_us, "conv_us": conv, "kernels": table}, f, indent=1)


if __name__ == "__main__":
    main()
