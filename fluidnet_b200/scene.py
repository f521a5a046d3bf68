"""The reference's 3-D demo (torch/fluid_net_3d_sim.lua:60-305) on the library: a plume rising from the floor of an
empty box, alone or around a voxelised arch or bunny, simulated for `numFrames` frames with the demo's settings, every
third density frame recorded to a `.vbox` file for Blender behind the running step (record.FrameRecorder), and the
obstacle geometry written once after frame 1.

    python -m fluidnet_b200.scene --res 128 --model data/models/myModel3D                  # the plume
    python -m fluidnet_b200.scene --scene arch --binvox voxels_demo/ --model ...           # the arch

The demo reads its obstacles from `../voxelizer/voxels_demo/Y91_arc_<modelRes>.binvox` and
`bunny.capped_<modelRes>.binvox`, with modelRes = 2^(floor(log2 res) - 1), half the grid (64 at 128^3).  Those files
do not ship with the reference: `--binvox` takes such a file, or a directory holding it under the demo's name.

Files, as the demo writes them (into --out-dir, by default the demo's render folder name):
  * density_output_<model>_dt0.1.vbox: the header says numFrames frames but only frames 3, 6, ... are written (the
    `.blend` scenes were made from files that look like this);
  * geom_output.vbox: the occupancy after frame 1 (tfluids.flagsToOccupancy), one frame;
  * geom_output_blender.vbox: the same with the six border planes zeroed, so the renderer can see inside.

With --slabs the domain is split into z-slabs, one rank per process (the library's slab step, tfl_slab_sim_step), and
every rank packs its planes of each recorded frame into rank 0's staging frame over peer memory
(record.SlabFrameRecorder); rank 0 writes the same files.  Under torchrun with more than one process --slabs is implied:

    torchrun --nproc-per-node 8 -m fluidnet_b200.scene --res 256 --sim-method jacobi
"""
import argparse
import math
import os
import time

import numpy as np

from . import formats
from .tfluids import CellType

SCENES = {"plume": "mushroom_cloud_render", "arch": "arch_render", "bunny": "bunny_render"}   # the demo's outDir
NUM_FRAMES = 768
OUTPUT_DECIMATION = 3
DENSITY_VAL = [1]
PLUME_RAD = 0.15
RES_RANGE = (16, 512)
# The z-slab margin the scene runs with unless told otherwise: planes a backward trace may reach.  Over the 768-frame
# 256^3 plume the longest trace (max |U| dt) measured 2.73 cells with 'jacobi' and 1.62 with a synthetic convnet model
# (DESIGN.md section 6a); a trace of t cells needs ceil(t) + 1 = 4, and 5 keeps one plane of headroom.
SLAB_MARGIN = 5


def model_res(res):
    """Resolution of the obstacle the demo loads: half the grid, rounded down to a power of two (:94)."""
    return int(math.pow(2, math.floor(math.log(res) / math.log(2)) - 1))


def binvox_name(scene, res):
    """File name the demo loads for `scene` at grid resolution `res` (:100-109)."""
    return {"arch": "Y91_arc_%d.binvox", "bunny": "bunny.capped_%d.binvox"}[scene] % model_res(res)


def lua_number(x):
    """A number as Lua's `..` prints it (%.14g): 0.1 -> '0.1', 2.0 -> '2'."""
    return "%.14g" % x


def density_filename(model_name, dt):
    """:159-160."""
    return "density_output_%s_dt%s.vbox" % (model_name, lua_number(dt))


def scene_mconf(res, sim_method="convnet", model_mconf=None):
    """The model's mconf with the demo's overrides (:73-87)."""
    if sim_method not in ("convnet", "jacobi", "pcg"):
        raise ValueError("simMethod must be 'convnet', 'jacobi' or 'pcg', not %r" % (sim_method,))
    mconf = dict(model_mconf or {})
    mconf.setdefault("normalizeInputThreshold", 1e-5)
    mconf.update(buoyancyScale=2.0 * (res / 128), gravityScale=0, dt=0.1, maccormackStrength=0.6, maxIter=34,
                 vorticityConfinementAmp=3, advectionMethod="maccormackOurs", simMethod=sim_method, is3D=True)
    return mconf


def empty_domain_flags(res, bnd=1):
    """tfluids.emptyDomain(FloatTensor(1, 1, res, res, res), true) on the host (tfluids/generic/tfluids.cc:136-166):
    obstacle cells on the bnd-thick border, fluid inside."""
    i = np.arange(res)
    edge = (i < bnd) | (i > res - 1 - bnd)
    border = edge[:, None, None] | edge[None, :, None] | edge[None, None, :]
    flags = np.where(border, np.float32(CellType.TypeObstacle), np.float32(CellType.TypeFluid))
    return np.ascontiguousarray(flags.reshape(1, 1, res, res, res), np.float32)


def obstacle_voxels(scene, res, binvox_path):
    """The demo's obstacle as a [res]^3 occupancy volume ([z][y][x]), or None for the plume alone (:92-119)."""
    if scene == "plume":
        return None
    if scene not in ("arch", "bunny"):
        raise ValueError("Bad conf.loadVoxelModel value")
    if binvox_path is None:
        raise ValueError("scene %r needs its binvox file (%s)" % (scene, binvox_name(scene, res)))
    if os.path.isdir(binvox_path):
        binvox_path = os.path.join(binvox_path, binvox_name(scene, res))
    vox = formats.load_binvox(binvox_path)["data"]
    formats.flip_diagonal(vox, 2)
    formats.flip_diagonal(vox, 0)
    offset = (0, -0.04 * res, 0) if scene == "arch" else (0.04 * res, 0, 0.04 * res)   # (x, y, z)
    return formats.pad_voxels_to_dims(res, res, res, vox, *offset)


def scene_flags(res, voxels=None):
    """Flags [1][1][res]^3: the empty domain, the occupancy copied into the interior [1, res - 2] as Obstacle / Fluid
    (:120-131)."""
    flags = empty_domain_flags(res)
    if voxels is not None:
        occ = np.asarray(voxels, np.float32).reshape(1, 1, res, res, res)[:, :, 1:res - 1, 1:res - 1, 1:res - 1]
        one = np.float32(1)
        flags[:, :, 1:res - 1, 1:res - 1, 1:res - 1] = (occ * np.float32(CellType.TypeObstacle) +
                                                        (one - occ) * np.float32(CellType.TypeFluid))
    return flags


def blender_geometry(occ):
    """The occupancy with its six border planes zeroed (:276-281)."""
    occ = occ.copy()
    for axis in range(3):
        idx = [slice(None)] * 3
        for end in (0, -1):
            idx[axis] = end
            occ[tuple(idx)] = 0
    return occ


def launcher_world():
    """(rank, world, local rank) of a torchrun launch, (0, 1, 0) without one."""
    env = os.environ
    return int(env.get("RANK", 0)), int(env.get("WORLD_SIZE", 1)), int(env.get("LOCAL_RANK", 0))


def check_slab_args(res, sim_method, world, margin):
    """The slab mode's refusals, before any rank touches a GPU; returns the margin (None -> SLAB_MARGIN)."""
    if sim_method == "pcg":
        raise ValueError("simMethod 'pcg' does not run on z-slabs: the IC(0) triangular solves of its preconditioner "
                         "sweep the whole domain in order (use 'jacobi' or 'convnet')")
    margin = SLAB_MARGIN if margin is None else int(margin)
    if margin < 2:
        raise ValueError("--margin must be >= 2 (got %d)" % margin)
    halo = 2 * margin + 2
    if world > 1 and res // world < halo:
        raise ValueError("%d planes over %d ranks give slabs of %d planes, thinner than the halo of %d (margin %d): "
                         "use fewer ranks or a smaller --margin" % (res, world, res // world, halo, margin))
    return margin


def scene_paths(out_dir, scene, model_name, dt, density_file=None):
    """The files the scene writes (the same in slab mode)."""
    out_dir = out_dir or SCENES[scene]
    return {"density": density_file or os.path.join(out_dir, density_filename(model_name, dt)),
            "geom": os.path.join(out_dir, "geom_output.vbox"),
            "geom_blender": os.path.join(out_dir, "geom_output_blender.vbox")}


def write_geometry(paths, res, flags):
    """The two geometry files from tfluids.flagsToOccupancy of `flags` (a device tensor)."""
    import torch
    from . import tfluids
    occ_t = torch.empty_like(flags)
    tfluids.flagsToOccupancy(flags, occ_t)
    occ = occ_t.cpu().numpy()[0, 0]
    with formats.VboxWriter(paths["geom"], res, 1) as w:
        w.write(occ)
    with formats.VboxWriter(paths["geom_blender"], res, 1) as w:
        w.write(blender_geometry(occ))


def run(res=128, scene="plume", sim_method="convnet", model=None, model_mconf=None, model_name="model",
        out_dir=None, binvox=None, num_frames=NUM_FRAMES, output_decimation=OUTPUT_DECIMATION, slots=3,
        density_file=None, log=print, slabs=False, margin=None, world=None, rank=None):
    """Simulate the scene and write its files; returns {'density', 'geom', 'geom_blender': paths,
    'ms_per_frame': host time per frame excluding frame 1 (None for a single frame), 'frames_written': n}.
    slabs: run on z-slabs (run_slabs), one rank per process; implied when the launcher's WORLD_SIZE > 1."""
    if not RES_RANGE[0] <= res <= RES_RANGE[1]:
        raise ValueError("res must lie in [%d, %d] (the demo's range), got %d" % (RES_RANGE + (res,)))
    if sim_method == "convnet" and model is None:
        raise ValueError("simMethod 'convnet' needs a model")
    env_rank, env_world, _ = launcher_world()
    world = env_world if world is None else int(world)
    rank = env_rank if rank is None else int(rank)
    if slabs or world > 1:
        margin = check_slab_args(res, sim_method, world, margin)
    mconf = scene_mconf(res, sim_method, model_mconf)
    if model is not None:
        mconf["normalizeInputThreshold"] = float(model.threshold)
    flags_np = scene_flags(res, obstacle_voxels(scene, res, binvox))
    paths = scene_paths(out_dir, scene, model_name, mconf["dt"], density_file)
    if rank == 0:
        os.makedirs(os.path.dirname(paths["geom"]) or ".", exist_ok=True)
        log("running simulation at resolution %d^3 (%s, simMethod %s), %d frames, saving every %d"
            % (res, scene, sim_method, num_frames, output_decimation))
    if slabs or world > 1:
        return run_slabs(res, mconf, model, flags_np, paths, num_frames, output_decimation, slots, margin, rank, world,
                         log)
    import torch
    from . import record, simulate, tfluids

    stream = torch.cuda.Stream()          # a step graph cannot be captured on the legacy default stream
    with torch.cuda.stream(stream):
        def zeros(c):
            return torch.zeros(1, c, res, res, res, dtype=torch.float32, device="cuda")
        batch = {"pDiv": zeros(1), "UDiv": zeros(3), "flags": torch.from_numpy(flags_np).cuda(), "density": zeros(1)}
        simulate.createPlumeBCs(batch, DENSITY_VAL, 1.0 * (res / 128), PLUME_RAD)
        rec = record.FrameRecorder((res, res, res), slots)
        graph = None
        t0 = None
        written = 0
        try:
            with formats.VboxWriter(paths["density"], res, num_frames) as dens:
                for i in range(1, num_frames + 1):
                    if i == 2:
                        stream.synchronize()      # frame 1 (and the graph capture) is not timed
                        t0 = time.perf_counter()
                    if graph is not None:
                        graph.launch()
                    else:
                        simulate.simulate_fused(None, mconf, batch, model)
                    if i == 1:
                        write_geometry(paths, res, batch["flags"])
                        graph = simulate.StepGraph(mconf, batch, model)
                    if i % output_decimation == 0:
                        rec.record(batch["density"], dens)
                        written += 1
                    rec.drain(dens)
                rec.drain(dens, wait=True)
            stream.synchronize()
            t1 = time.perf_counter()
            if graph is not None and sim_method == "pcg":
                graph.pcg_status()        # raises what the reference's solve would have (a NaN residual, ...)
        finally:
            rec.close()
            if graph is not None:
                graph.close()
    ms = None if t0 is None else 1000.0 * (t1 - t0) / (num_frames - 1)
    log("All done!")
    if ms is not None:
        log("Processing time: %.4f ms per frame" % ms)
    return dict(paths, ms_per_frame=ms, frames_written=int(written))


def run_slabs(res, mconf, model, flags_np, paths, num_frames, output_decimation, slots, margin, rank, world, log):
    """run() on z-slabs: rank `rank` of `world` steps its slab with the library's slab step (NativeSlabSimulator) and
    captures every `output_decimation`-th density frame into a SlabFrameRecorder; rank 0 writes the files.  Every rank
    holds the global flags and BCs.  Without peer memory the frames are gathered synchronously (and the log says so).
    After the run the trace faults of all ranks are summed, and a non-zero count raises."""
    import torch
    import torch.distributed as dist
    from . import simulate
    from ._lib import TflError
    from .slab import NativeSlabSimulator

    _, _, local = launcher_world()
    if world > 1 and not dist.is_initialized():
        torch.cuda.set_device(local)
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", local))
    device = torch.device("cuda", torch.cuda.current_device())
    zeros = lambda c: torch.zeros(1, c, res, res, res, dtype=torch.float32)    # noqa: E731
    batch = {"pDiv": zeros(1), "UDiv": zeros(3), "flags": torch.from_numpy(flags_np), "density": zeros(1)}
    simulate.createPlumeBCs(batch, DENSITY_VAL, 1.0 * (res / 128), PLUME_RAD)     # on the host, as the whole-grid scene
    stream = torch.cuda.Stream(device)
    written, t0, rec, dens = 0, None, None, None
    with torch.cuda.stream(stream):
        sim = NativeSlabSimulator(batch, mconf, None, device, rank, world, margin, model=model)
        try:
            try:
                rec = sim.frame_recorder(slots)
                transport = "peer memory" if world > 1 else "one rank"
            except TflError as e:
                transport = "a synchronous gather (%s)" % e
            if rank == 0:
                log("z-slabs: %d rank(s), margin %d, halos over %s, frames through %s"
                    % (world, margin, sim.halo_transport, transport))
                dens = formats.VboxWriter(paths["density"], res, num_frames)
            for i in range(1, num_frames + 1):
                if i == 2:
                    stream.synchronize()      # frame 1 is not timed
                    t0 = time.perf_counter()
                sim.step()
                if i == 1 and rank == 0:
                    write_geometry(paths, res, batch["flags"].to(device))
                if i % output_decimation == 0:
                    if rec is not None:
                        sim.record(rec, dens)
                    else:
                        frame = sim.gather("density")
                        if rank == 0:
                            dens.write(frame.numpy())
                    written += 1
                if rec is not None:
                    rec.drain(dens)
            if rec is not None:
                rec.drain(dens, wait=True)
            stream.synchronize()
            t1 = time.perf_counter()
            try:
                sim.check()
            except RuntimeError as e:
                raise RuntimeError("%s (the scene's --margin, now %d)" % (e, margin)) from None
        finally:
            if dens is not None:
                dens.close()
            if rec is not None:
                rec.close()
            sim.close()
    ms = None if t0 is None else 1000.0 * (t1 - t0) / (num_frames - 1)
    if rank == 0:
        log("All done!")
        if ms is not None:
            log("Processing time: %.4f ms per frame" % ms)
    return dict(paths, ms_per_frame=ms, frames_written=int(written))


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--res", type=int, default=128, help="grid resolution, 16 .. 512 (the demo: a power of two)")
    ap.add_argument("--scene", default="plume", choices=sorted(SCENES))
    ap.add_argument("--binvox", help="the obstacle's .binvox file, or a directory holding the demo's file name")
    ap.add_argument("--sim-method", default="convnet", choices=["convnet", "jacobi", "pcg"])
    ap.add_argument("--model", help="a model saved by the reference (its _mconf.bin beside it)")
    ap.add_argument("--synthetic-model", action="store_true", help="a seeded synthetic 3-D model instead")
    ap.add_argument("--frames", type=int, default=NUM_FRAMES)
    ap.add_argument("--decimation", type=int, default=OUTPUT_DECIMATION)
    ap.add_argument("--slots", type=int, default=3, help="pinned host frames in the recorder's ring")
    ap.add_argument("--out-dir")
    ap.add_argument("--density-filename", help="the density file's path (default: the demo's name in --out-dir)")
    ap.add_argument("--slabs", action="store_true",
                    help="run on z-slabs, one rank per process (implied under torchrun with more than one process)")
    ap.add_argument("--margin", type=int, default=None,
                    help="z-slab margin: planes a backward trace may reach (default %d, from the measured plume)"
                         % SLAB_MARGIN)
    args = ap.parse_args(argv)
    rank, world, local = launcher_world()
    if args.slabs or world > 1:
        check_slab_args(args.res, args.sim_method, world, args.margin)
        if world > 1:
            import torch
            torch.cuda.set_device(local)          # the model below lives on this rank's GPU
    model, model_mconf, name = None, None, "none"
    if args.model:
        from .model import ProjectionModel
        model, model_mconf = ProjectionModel.from_reference_file(args.model)
        name = os.path.basename(args.model.rstrip("/"))
    elif args.synthetic_model:
        from . import synth
        from .model import ProjectionModel
        model = ProjectionModel(synth.make_model(True)["layers"], True)
        name = "synthetic"
    run(args.res, args.scene, args.sim_method, model, model_mconf, name, args.out_dir, args.binvox, args.frames,
        args.decimation, args.slots, args.density_filename, print if rank == 0 else (lambda *a: None), args.slabs,
        args.margin)


if __name__ == "__main__":
    main()
