"""What recording density frames costs a z-slab run, what k_pack_vbox costs, and how long the scene's traces get.

    python tests/dbg_slab_record_rate.py [--steps-128 300] [--steps-256 90] [--reps 3] [--margin-frames 768]
    python tests/dbg_slab_record_rate.py --pack-only          # k_pack_vbox alone

* Step rate: the library's slab step (NativeSlabSimulator, one rank, simMethod 'jacobi', the scene's plume) at 128^3
  and 256^3 in four arms run alternately, `reps` times each, every run from the same state: no recording; the slab
  recorder every 3rd frame; every frame; and a synchronous gather (tfl_slab_sim_download) every 3rd frame.  Frames go
  to a `.vbox` writer on os.devnull.  The number is the host clock around `steps` steps and the final synchronise.
* Pack time: k_pack_vbox alone through the whole-grid recorder and the world-1 slab recorder, CUDA events around 100
  captures, each after a 256 MB L2 flush and each frame taken before the next, against its 8 B/cell bound at the
  H100 data sheet's 3.35 TB/s.
* Trace length: the largest max|U| dt over the single-GPU scene at 256^3 (plume; jacobi and a seeded synthetic
  convnet model), the step replayed from its graph as the scene does.  The scene's z-slab margin default rests on it.
Prints the card's name, power limit and max SM clock read in the same run, then one JSON line.
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

from fluidnet_b200 import _lib, formats, record, scene, simulate, synth      # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown (%s)" % q.stderr.strip()


def plume_batch(n):
    z = lambda c: torch.zeros(1, c, n, n, n)       # noqa: E731
    batch = {"pDiv": z(1), "UDiv": z(3), "flags": torch.from_numpy(scene.scene_flags(n)), "density": z(1)}
    simulate.createPlumeBCs(batch, [1], n / 128, 0.15)
    return batch


def step_rate(n, arm, steps, batch):
    from fluidnet_b200.slab import NativeSlabSimulator
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        sim = NativeSlabSimulator(batch, scene.scene_mconf(n, "jacobi"), None, torch.device("cuda", 0), 0, 1,
                                  scene.SLAB_MARGIN)
        rec = sim.frame_recorder(3) if arm.startswith("recorder") else None
        every = 1 if arm == "recorder_every_frame" else 3
        with formats.VboxWriter(os.devnull, n, steps) as w:
            sim.step()
            stream.synchronize()
            t0 = time.perf_counter()
            for i in range(1, steps + 1):
                sim.step()
                if arm != "none" and i % every == 0:
                    if rec is not None:
                        sim.record(rec, w)
                    else:
                        w.write(sim.gather("density").numpy())
                if rec is not None:
                    rec.drain(w)
            if rec is not None:
                rec.drain(w, wait=True)
            stream.synchronize()
            t1 = time.perf_counter()
        if rec is not None:
            rec.close()
        sim.close()
    return steps / (t1 - t0)


def pack_time(n, slab):
    """µs per k_pack_vbox (CUDA events around each capture, after an L2 flush)."""
    flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device="cuda")
    d = torch.rand(1, 1, n, n, n, device="cuda")
    stream = torch.cuda.current_stream()
    rec = record.SlabFrameRecorder((n, n, n), 0, 1, 1) if slab else record.FrameRecorder((n, n, n), 1)
    cap = (lambda: rec.capture(d, 0)) if slab else (lambda: rec.capture(d))
    times = []
    for i in range(110):
        flush.fill_(0.0)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        cap()
        b.record(stream)
        rec.take(wait=True)
        rec.release()
        if i >= 10:
            times.append(a.elapsed_time(b) * 1000.0)
    rec.close()
    us = float(np.median(times))
    bound = 8.0 * n ** 3 / 3.35e12 * 1e6
    return {"us": round(us, 2), "bound_us": round(bound, 2), "TB_per_s": round(8.0 * n ** 3 / us / 1e6, 3)}


def longest_trace(n, frames, sim_method):
    from fluidnet_b200.model import ProjectionModel
    model = ProjectionModel(synth.make_model(True)["layers"], True) if sim_method == "convnet" else None
    mconf = scene.scene_mconf(n, sim_method)
    if model is not None:
        mconf["normalizeInputThreshold"] = float(model.threshold)
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        z = lambda c: torch.zeros(1, c, n, n, n, device="cuda")      # noqa: E731
        batch = {"pDiv": z(1), "UDiv": z(3), "flags": torch.from_numpy(scene.scene_flags(n)).cuda(), "density": z(1)}
        simulate.createPlumeBCs(batch, [1], n / 128, 0.15)
        simulate.simulate_fused(None, mconf, batch, model)
        graph = simulate.StepGraph(mconf, batch, model)
        peaks = []
        for i in range(2, frames + 1):
            graph.launch()
            peaks.append(batch["UDiv"].abs().max())
        graph.close()
        vals = torch.stack(peaks).cpu().numpy() * mconf["dt"]
    worst, at = float(vals.max()), int(vals.argmax()) + 2
    return {"max_u_dt_cells": round(worst, 4), "at_frame": at, "frames": frames}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps-128", type=int, default=300)
    ap.add_argument("--steps-256", type=int, default=90)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--margin-frames", type=int, default=768)
    ap.add_argument("--pack-only", action="store_true")
    ap.add_argument("--out")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this measurement needs a GPU"
    res = {"card": card(), "lib": _lib.LIB_PATH}
    print(res["card"], res["lib"], flush=True)
    res["pack"] = {}
    for n in (128, 256):
        res["pack"][str(n)] = {"whole_grid": pack_time(n, False), "slab_world1": pack_time(n, True)}
        print("pack", n, json.dumps(res["pack"][str(n)]), flush=True)
    if not args.pack_only:
        arms = ["none", "recorder_every_3rd", "recorder_every_frame", "sync_gather_every_3rd"]
        res["rate"] = {}
        for n, steps in ((128, args.steps_128), (256, args.steps_256)):
            batch = plume_batch(n)
            rates = {a: [] for a in arms}
            step_rate(n, "none", 10, batch)                    # warm-up
            for r in range(args.reps):
                for a in arms:
                    rates[a].append(round(step_rate(n, a, steps, batch), 1))
                    print(n, a, "rep", r, rates[a][-1], "steps/s", flush=True)
            res["rate"][str(n)] = {"steps": steps, "steps_per_s": rates}
        res["trace"] = {m: longest_trace(256, args.margin_frames, m) for m in ("jacobi", "convnet")}
        print("trace", json.dumps(res["trace"]), flush=True)
    print(json.dumps(res), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
