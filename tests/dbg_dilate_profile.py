"""Dilated-bank projection models (banksType 'dilate') at the bench's 128^3 step, beside the single-bank model: each
model's step is replayed from a CUDA graph (simulate.StepGraph) with the L2 flushed in between, timed with CUDA
events, then profiled per kernel under torch.profiler.  Every model in 3xTF32, TF32 and fp32.  Prints the card, its
power limit and SM clock, steps/s, the convolution kernels' us per step, and the us per step of the bank plumbing:
the phase copy / re-zeroing on the tensor cores, the full-resolution 'add' join on the fp32 path.

    python tests/dbg_dilate_profile.py [--grid 128] [--steps 20]"""
import argparse
import os
import sys
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from dbg_step_profile import card  # noqa: E402

CONFIGS = [("default", None, "tf32x3"), ("default", None, "tf32"), ("default", None, "fp32")] + [
    (name, bk, mode) for mode in ("tf32x3", "tf32", "fp32")
    for name, bk in (("N2 concat", (2, "concat")), ("N3 concat", (3, "concat")), ("N2 add", (2, "add")))]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--grid", type=int, default=128)
    ap.add_argument("--steps", type=int, default=20)
    args = ap.parse_args()

    import torch
    from torch.profiler import profile, ProfilerActivity
    import bench
    from fluidnet_b200 import simulate, synth, model as fmodel

    assert torch.cuda.is_available(), "the profile needs a CUDA device"
    torch.cuda.set_device(0)
    batch_np, mconf, _ = bench.make_problem(args.grid)
    info = card()
    print("card: %s, power limit %s, SM clock %s (max %s)" % (info.get("name"), info.get("power.limit"),
                                                             info.get("clocks.sm"), info.get("clocks.max.sm")))
    print("%-10s %-7s %9s %12s %12s" % ("model", "mode", "steps/s", "conv us/step", "banks us/step"))
    stream = torch.cuda.Stream()
    flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device="cuda")
    for name, bk, mode in CONFIGS:
        banks = None if bk is None else {"num": bk[0], "split_stage": 1, "join_stage": 3, "aggregate": bk[1],
                                         "type": "dilate"}
        mnp = synth.make_model(True, banks=banks)
        with torch.cuda.stream(stream):
            gb = {k: torch.from_numpy(v.copy()).cuda() for k, v in batch_np.items()}
            gm = fmodel.ProjectionModel(mnp["layers"], True, banks=banks)
            gm.set_mode(mode)
            for _ in range(3):
                simulate.simulate_fused(None, mconf, gb, gm)
            graph = simulate.StepGraph(mconf, gb, gm)
            for _ in range(3):
                graph.launch()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ms = 0.0
            for _ in range(args.steps):
                flush.fill_(0.0)
                e0.record(stream)
                graph.launch()
                e1.record(stream)
                e1.synchronize()
                ms += e0.elapsed_time(e1)
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(args.steps):
                    flush.fill_(0.0)
                    graph.launch()
                stream.synchronize()
            graph.close()
        tot = defaultdict(float)
        for ev in prof.events():
            if ev.device_type == torch.autograd.DeviceType.CUDA:
                tot[ev.name] += ev.device_time / args.steps
        conv = sum(v for k, v in tot.items() if "k_conv3_tc" in k or "k_conv_direct" in k or "k_conv_any" in k)
        join = sum(v for k, v in tot.items() if "k_bank_join" in k or "k_tc_phase" in k)
        print("%-10s %-7s %9.1f %12.1f %12.1f" % (name, mode, 1000.0 * args.steps / ms, conv, join))
        del gm, gb
    print("SM clock after: %s" % card().get("clocks.sm"))


if __name__ == "__main__":
    main()
