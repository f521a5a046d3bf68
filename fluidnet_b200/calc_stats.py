"""The reference's model evaluation, torch.calcStats (torch/lib/calc_stats.lua:52-118), on the library: batches of
start frames are stepped `nSteps - 1` times, and after the start frame and every step each sample's divergence norm
(`div[i]:norm()`) is recorded -- the divergence-versus-time table of the paper.

    python -m fluidnet_b200.calc_stats --model data/models/myModel3D --steps 128 --batch 16 --out stats.csv tr/*.bin
    python -m fluidnet_b200.calc_stats --synthetic 32 --res 64 --seed 1 --synthetic-model --batch 8 --out stats.csv

Start frames are Manta `.bin` dumps (formats.load_manta_file; every file must have the same shape and dimensionality)
or seeded synthetic frames (synth: sphere + slab flags, a smooth velocity, p = 0 and a density).  As in the reference,
p and U restart from the frame, the model's mconf runs with gravityScale = 0 (calc_stats.lua:105), and no boundary
conditions are set.  --sim-method runs the 'jacobi' or 'pcg' solve instead of the model (maxIter 34, as
fluid_net_train.lua's CalcAndDumpStats sets it).

Frames are stepped --batch at a time as one [b][c][z][y][x] batch (conf.batchSize; the last batch may be shorter).  Per
batch the step monitor (monitor.StepMonitor) records the start frame, step 2 runs through simulate_fused, and steps 3..N
replay a StepGraph of it; the monitor records after every step on the device and the host only takes a record when the
ring is full, so no step waits for the host.  3-D convnet batches take the fused step; 2-D frames run the operator path.

The CSV has one row per (sample, step): sample (0-based position in the frame list), source (file name or
synthetic:<seed>), step (1 = the start frame), div_norm, div_max (max |div|) and u_max_dt (max |U| dt, the longest
trace in cells).  The log gives the mean div_norm of every step and the largest u_max_dt.
"""
import argparse
import os

import numpy as np

from . import formats, monitor, scene

COLUMNS = ("sample", "source", "step", "div_norm", "div_max", "u_max_dt")
MONITOR_CAPACITY = 64
# lib/default_conf.lua's newModel settings that the step reads, for a model without an mconf of its own
DEFAULT_MCONF = dict(dt=0.1, advectionMethod="maccormack", maccormackStrength=0.75, buoyancyScale=0,
                     gravityScale=0, vorticityConfinementAmp=0.0, simMethod="convnet")


class Frame:
    """One start frame: [1][c][z][y][x] float32 arrays and where it came from."""

    def __init__(self, source, p, U, flags, density, is3d):
        self.source, self.p, self.U, self.flags, self.density, self.is3d = source, p, U, flags, density, bool(is3d)

    @property
    def shape(self):
        return tuple(self.flags.shape[2:])


def load_frames(paths):
    """Manta frames from `paths`; every one must have the first one's shape and dimensionality."""
    frames = []
    for path in paths:
        p, U, flags, density, is3d = formats.load_manta_file(path)
        f = Frame(os.path.basename(path), p, U, flags, density, is3d)
        if frames and (f.shape != frames[0].shape or f.is3d != frames[0].is3d):
            raise ValueError("%s is a %s %s frame, but %s is a %s %s frame: a run takes frames of one shape"
                             % (path, "x".join(map(str, f.shape[::-1])), "3-D" if f.is3d else "2-D", frames[0].source,
                                "x".join(map(str, frames[0].shape[::-1])), "3-D" if frames[0].is3d else "2-D"))
        frames.append(f)
    return frames


def synthetic_frames(count, res, seed, is3d=True):
    """`count` seeded frames at res^3 (res^2 in 2-D): sphere + slab flags, a smooth velocity (seed + i), p = 0 and a
    density (seed + i)."""
    from . import synth
    nz = res if is3d else 1
    flags = synth.make_flags(res, res, nz, is3d, 1, geometry=True)
    out = []
    for i in range(count):
        U = synth.make_smooth_velocity(flags, is3d, seed=seed + i)
        d = synth.make_density(flags, seed=seed + i)
        out.append(Frame("synthetic:%d" % (seed + i), np.zeros_like(flags), U, flags.copy(), d, is3d))
    return out


def group(frames, batch):
    """Consecutive batches of at most `batch` frames: [(first sample index, [frames])]."""
    if batch < 1:
        raise ValueError("--batch must be >= 1 (got %d)" % batch)
    return [(i, frames[i:i + batch]) for i in range(0, len(frames), batch)]


def eval_mconf(model_mconf=None, sim_method=None):
    """The model's mconf (DEFAULT_MCONF without one) as calcStats runs it: gravityScale = 0, maxIter = 34, and
    simMethod replaced by `sim_method` when given."""
    mconf = dict(DEFAULT_MCONF)
    mconf.update(model_mconf or {})
    mconf["gravityScale"] = 0
    mconf["maxIter"] = 34
    if sim_method is not None:
        mconf["simMethod"] = sim_method
    if mconf.get("simMethod", "convnet") not in ("convnet", "jacobi", "pcg"):
        raise ValueError("simMethod must be 'convnet', 'jacobi' or 'pcg', not %r" % (mconf["simMethod"],))
    return mconf


def _batch_tensors(frames):
    import torch
    cat = lambda name: torch.from_numpy(np.concatenate([getattr(f, name) for f in frames])).cuda()   # noqa: E731
    return {"pDiv": cat("p"), "UDiv": cat("U"), "flags": cat("flags"), "density": cat("density")}


def run_batch(frames, mconf, model, steps):
    """Steps one batch of frames on the current CUDA stream (not the legacy default one) -> [nb][steps][3] float64
    (div_norm, div_max, u_max) after the start frame and after each step."""
    from . import simulate
    batch = _batch_tensors(frames)
    mconf = dict(mconf, is3D=frames[0].is3d)
    nb = len(frames)
    out = np.full((nb, steps, 3), np.nan)
    mon = monitor.StepMonitor(None, batch, MONITOR_CAPACITY)
    graph = None

    def keep(rec):
        out[:, rec[0]] = rec[1]

    try:
        for j in range(steps):                # j = 0: the start frame, then one step before each record
            if j == 1:
                simulate.simulate_fused(None, mconf, batch, model)
            elif j > 1:
                if graph is None:
                    graph = simulate.StepGraph(mconf, batch, model)
                graph.launch()
            if mon.full:
                keep(mon.take())
            mon.record(batch)
        if graph is not None and mconf.get("simMethod") == "pcg":
            graph.pcg_status()               # raises what the reference's solve would have
        for rec in mon.drain(wait=True):
            keep(rec)
    finally:
        mon.close()
        if graph is not None:
            graph.close()
    return out


def run(frames, mconf, model, steps, batch, log=print):
    """Every frame stepped in batches of `batch` -> rows (sample, source, step, div_norm, div_max, u_max_dt)."""
    import torch
    if steps < 1:
        raise ValueError("--steps must be >= 1 (got %d)" % steps)
    if not frames:
        raise ValueError("no start frames")
    if mconf.get("simMethod", "convnet") == "convnet" and model is None:
        raise ValueError("simMethod 'convnet' needs a model")
    if model is not None and model.is3D != frames[0].is3d:
        raise ValueError("a %s model cannot step %s frames" % ("3-D" if model.is3D else "2-D",
                                                              "3-D" if frames[0].is3d else "2-D"))
    mconf = dict(mconf)
    if model is not None:
        mconf["normalizeInputThreshold"] = float(model.threshold)
    rows = []
    stream = torch.cuda.Stream()              # a step graph cannot be captured on the legacy default stream
    with torch.cuda.stream(stream):
        for first, part in group(frames, batch):
            vals = run_batch(part, mconf, model, steps)
            for b, f in enumerate(part):
                for j in range(steps):
                    dn, dm, um = vals[b, j]
                    rows.append((first + b, f.source, j + 1, dn, dm, um * mconf["dt"]))
    summarize(rows, steps, log)
    return rows


def summarize(rows, steps, log=print):
    """Logs the mean div_norm of every step and the largest u_max_dt; returns (means, peak)."""
    means = []
    for j in range(1, steps + 1):
        v = [r[3] for r in rows if r[2] == j]
        means.append(sum(v) / len(v))
    peak = 0.0
    for r in rows:
        peak = monitor._nanmax(peak, r[5])
    log("mean div_norm per step: " + " ".join("%d:%.6g" % (j + 1, m) for j, m in enumerate(means)))
    log("%d samples, %d steps; largest max|U| dt: %.4f cells" % (len({r[0] for r in rows}), steps, peak))
    return means, peak


def write_csv(path, rows):
    os.makedirs(os.path.dirname(path) or ".", exist_ok=True)
    with open(path, "w") as f:
        f.write(",".join(COLUMNS) + "\n")
        for sample, source, step, dn, dm, ud in rows:
            if "," in source or "\n" in source:
                raise ValueError("source %r cannot go into the CSV" % source)
            f.write("%d,%s,%d,%s,%s,%s\n" % (sample, source, step, scene.csv_float(dn), scene.csv_float(dm),
                                             scene.csv_float(ud)))


def read_csv(path):
    with open(path) as f:
        head = f.readline().strip().split(",")
        if tuple(head) != COLUMNS:
            raise ValueError("%s is not a calc_stats file (header %r)" % (path, head))
        return [(int(r[0]), r[1], int(r[2]), float(r[3]), float(r[4]), float(r[5]))
                for r in (ln.rstrip("\n").split(",") for ln in f) if r[0]]


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("frames", nargs="*", help="Manta .bin start frames (all of one shape)")
    ap.add_argument("--synthetic", type=int, metavar="COUNT", help="COUNT seeded synthetic frames instead of files")
    ap.add_argument("--res", type=int, default=64, help="grid size of the synthetic frames")
    ap.add_argument("--seed", type=int, default=1, help="seed of the first synthetic frame")
    ap.add_argument("--model", help="a model saved by the reference (its _mconf.bin beside it)")
    ap.add_argument("--synthetic-model", action="store_true", help="a seeded synthetic model instead")
    ap.add_argument("--sim-method", choices=["convnet", "jacobi", "pcg"],
                    help="the projection to run (default: the model's simMethod)")
    ap.add_argument("--steps", type=int, default=128, help="nSteps: the start frame counts as step 1 (default 128)")
    ap.add_argument("--batch", type=int, default=16, help="frames stepped together (conf.batchSize, default 16)")
    ap.add_argument("--out", default="calc_stats.csv", help="the CSV file")
    args = ap.parse_args(argv)
    if bool(args.frames) == (args.synthetic is not None):
        ap.error("give either Manta frames or --synthetic COUNT")
    if args.synthetic is not None and (args.synthetic < 1 or args.res < 4):
        ap.error("--synthetic needs COUNT >= 1 and --res >= 4")
    if args.model and args.synthetic_model:
        ap.error("--model and --synthetic-model exclude each other")
    if args.steps < 1 or args.batch < 1:
        ap.error("--steps and --batch must be >= 1")
    return args


def main(argv=None):
    args = parse_args(argv)
    frames = synthetic_frames(args.synthetic, args.res, args.seed) if args.synthetic is not None \
        else load_frames(args.frames)
    model, model_mconf = None, None
    if args.model:
        from .model import ProjectionModel
        model, model_mconf = ProjectionModel.from_reference_file(args.model)
    elif args.synthetic_model:
        from . import synth
        from .model import ProjectionModel
        model = ProjectionModel(synth.make_model(frames[0].is3d)["layers"], frames[0].is3d)
    mconf = eval_mconf(model_mconf, args.sim_method)
    print("calc_stats: %d frames of %s, simMethod %s, %d steps, batches of %d"
          % (len(frames), "x".join(map(str, frames[0].shape[::-1])), mconf["simMethod"], args.steps, args.batch))
    rows = run(frames, mconf, model, args.steps, args.batch)
    write_csv(args.out, rows)
    print("wrote %d rows to %s" % (len(rows), args.out))


if __name__ == "__main__":
    main()
