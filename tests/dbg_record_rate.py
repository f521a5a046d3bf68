"""What recording density frames costs the replayed step (fluidnet_b200/record.py).

    python tests/dbg_record_rate.py [--steps-128 600] [--steps-256 120] [--reps 3] [--out results.json]

At 128^3 and 256^3 (the bench's plume problem, the step replayed from a CUDA graph), steps/s in four arms run
alternately, `reps` times each: no recording; the recorder every 3rd frame; the recorder every frame; and the
reference's way, a synchronous `permute(3, 2, 1):contiguous()` download every 3rd frame.  Frames go to a `.vbox`
writer on os.devnull: the host's write path without the disk.  Each arm starts from the same state and its time is the
host clock around `steps` launches and the final stream synchronise.  Also times k_pack_vbox alone (CUDA events around 200 captures, each frame taken
before the next, with the L2 warm and after a 256 MB flush) and one pinned device-to-host copy of a frame, and prints the
card's name, power limit and max SM clock.
"""
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

from fluidnet_b200 import formats, record, scene, simulate, synth          # noqa: E402
from fluidnet_b200.model import ProjectionModel                             # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown (%s)" % q.stderr.strip()


def problem(n, net):
    flags = synth.make_flags(n, n, n, True, nb=1, geometry=True)
    batch = {"pDiv": np.zeros_like(flags), "UDiv": synth.make_smooth_velocity(flags, True, amp=2.0), "flags": flags,
             "density": synth.make_density(flags)}
    gb = {k: torch.from_numpy(v.copy()).cuda() for k, v in batch.items()}
    simulate.createPlumeBCs(gb, [1.0], n / 128.0, 0.15)
    mconf = scene.scene_mconf(n)
    mconf["normalizeInputThreshold"] = float(net.threshold)
    return gb, mconf


def run_arm(arm, graph, gb, start, rec, sink, steps, stream):
    for k, v in start.items():                  # every arm replays the same steps: the step's cost grows as the plume
        gb[k].copy_(v)                          # accelerates, so an evolving state would favour the earlier arms
    d = gb["density"]
    stream.synchronize()
    t0 = time.perf_counter()
    for i in range(1, steps + 1):
        graph.launch()
        if arm == "recorder_every_3rd" and i % 3 == 0:
            rec.record(d, sink)
        elif arm == "recorder_every_frame":
            rec.record(d, sink)
        elif arm == "sync_permute_every_3rd" and i % 3 == 0:
            sink.write_packed(d[0, 0].permute(2, 1, 0).contiguous().cpu().numpy())
        if rec is not None:
            rec.drain(sink)
    if rec is not None:
        rec.drain(sink, wait=True)
    stream.synchronize()
    return steps / (time.perf_counter() - t0)


def pack_times(n, stream, iters=200):
    d = torch.rand(1, 1, n, n, n, device="cuda")
    flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device="cuda")
    out = {}
    with record.FrameRecorder(d.shape, slots=2) as rec:
        for label, flushed in (("warm_l2", False), ("flushed_l2", True)):
            ms = []
            for _ in range(iters):
                if flushed:
                    flush.fill_(0.0)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                rec.capture(d)
                e1.record(stream)
                rec.take(wait=True)
                rec.release()
                ms.append(e0.elapsed_time(e1))
            ms = float(np.median(ms))
            out[label] = {"ms_median": ms, "GB_per_s": 8.0 * n ** 3 / (ms * 1e6)}
    pinned = torch.empty(n ** 3, dtype=torch.float32).pin_memory()
    src = torch.rand(n ** 3, device="cuda")
    ms = []
    for _ in range(20):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        pinned.copy_(src, non_blocking=True)
        e1.record(stream)
        stream.synchronize()
        ms.append(e0.elapsed_time(e1))
    out["d2h_copy"] = {"ms_median": float(np.median(ms)), "GB_per_s": 4.0 * n ** 3 / (float(np.median(ms)) * 1e6)}
    out["algorithmic_MB"] = 8.0 * n ** 3 / 1e6
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps-128", type=int, default=600)
    ap.add_argument("--steps-256", type=int, default=120)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", help="also write the results as JSON to this file")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this measurement needs a GPU"
    torch.cuda.set_device(0)
    res = {"card": card(), "torch": torch.__version__, "grids": {}}
    print(res["card"], flush=True)
    arms = ["none", "recorder_every_3rd", "recorder_every_frame", "sync_permute_every_3rd"]
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        net = ProjectionModel(synth.make_model(True)["layers"], True)
        for n, steps in ((128, args.steps_128), (256, args.steps_256)):
            gb, mconf = problem(n, net)
            simulate.simulate_fused(None, mconf, gb, net)
            graph = simulate.StepGraph(mconf, gb, net)
            start = {k: gb[k].clone() for k in ("pDiv", "UDiv", "density")}
            rates = {a: [] for a in arms}
            with record.FrameRecorder(gb["density"].shape, slots=3) as rec, \
                    formats.VboxWriter(os.devnull, n, 0) as sink:
                for a in arms:                                   # warm-up, untimed
                    run_arm(a, graph, gb, start, rec if a.startswith("recorder") else None, sink, 6, stream)
                for r in range(args.reps):
                    for a in arms:
                        rates[a].append(run_arm(a, graph, gb, start, rec if a.startswith("recorder") else None, sink,
                                                steps, stream))
                        print(n, a, "rep", r, "%.1f steps/s" % rates[a][-1], flush=True)
            graph.close()
            del gb
            torch.cuda.empty_cache()
            res["grids"][str(n)] = {"steps": steps, "steps_per_s": rates, "pack": pack_times(n, stream)}
            print(json.dumps(res["grids"][str(n)]["pack"]), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
