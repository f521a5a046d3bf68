"""The batched fused step (tfl_simulate_step at nb > 1) on every tensor-core model, and the launch grid's limits.

Models, each in 3xTF32 and TF32: the default one; 'mres' banks N = 2 concat and N = 3 add; 'dilate' banks N = 2 concat
and N = 3 add on grids 2 and 4 do not divide; batch normalization with batch statistics and with running statistics;
batch statistics with relu6 (the first stage scaled so that values cross 6); relu6 with 'mres' N = 2 concat.

Scenes: nb = 2 and 3 entries of their own flags (one with fluid on its x and z faces, so that the planes a quad block
shares between two entries carry velocity into the input scale's sums), velocity amplitude (one entry at rest),
density and plume BCs.  The shapes take the quad kernels with blocks straddling two entries (nb nz odd), the
per-voxel kernels (nx % 4 != 0) and a row wider than 128 (the box tensor-core convolution).

Three steps per case, each re-seeded from the GPU's state (as tests/test_gpu_step_paths.py does):
  (1) float64, per voxel: every voxel of p and U of every entry within the bound E of tests/network_bound.py on the
      scale interval (projection_reference of tests/test_gpu_cnn_network_f64.py, batches included); the largest
      err / E of each case is printed;
  (2) the operator sequence (simulate.simulate): density bit for bit, U and p within OPS_TOL with the same zero bits;
  (3) oracle.simulate with the network in float64: density bit for bit, U and p within MODE_TOL (TF32 with
      batch statistics: 1e-2, oracle_tol);
  (4) entries: for every model without batch statistics each entry equals its scene stepped alone (OPS_TOL, zero
      bits); with batch statistics changing entry 1 changes entry 0's p (and (2) holds for the coupled batch);
  (5) no trace fault.
A banked and a batch-statistics model replay a step graph bit for bit with in-place changes between replays;
test_fused_kernels_ran proves from torch.profiler's kernel names that every case ran the fused kernels it was meant to
(quad or per-voxel), and that the launch tally counts exactly what ran.  calc_stats with a batch-statistics model at
batch 3 writes the rows of a plain loop over the same batches.

Launch grid: CUDA allows 65535 blocks along gridDim.y and z, and the launchers put the batch's planes there
(check_launch_grid, fluidnet_b200/csrc/tfl_api_internal.h).  The largest batch make_geo accepts of an 8x8 grid (2-D:
nb = 65535; 3-D nz = 5: nb nz = 131070) runs the operator step, the fused step, a Jacobi solve with pTol > 0 and the
step monitor, every entry equal to the oracle on its prototype; one entry more is refused by name before anything is
launched, and the context steps a valid batch afterwards."""
import ctypes as C

import numpy as np
import pytest
import torch

import monitor_reference
import oracle
from cases import bits_equal, describe_diff
from fluidnet_b200 import synth
from fluidnet_b200.model import ProjectionModel
from network_bound import check, projection_reference, tc_covered
from scenes import banks, bn_model
from step_cases import (MODE_TOL, OPS_TOL, close_per_entry, plume_bcs, quad_dims, run_in_child, same_zero_bits,
                        takes_fused_path)

MCONF = oracle.default_mconf(dt=0.1, maccormackStrength=0.6, buoyancyScale=0.5, vorticityConfinementAmp=3.0,
                             simMethod="convnet")
JACOBI = oracle.default_mconf(dt=0.1, maccormackStrength=0.6, buoyancyScale=0.5, vorticityConfinementAmp=3.0,
                              simMethod="jacobi", maxIter=12)


MODELS = {
    "default": lambda: synth.make_model(True),
    "mres-n2-concat": lambda: synth.make_model(True, banks=banks(2, "concat", "mres")),
    "mres-n3-add": lambda: synth.make_model(True, banks=banks(3, "add", "mres")),
    "dilate-n2-concat": lambda: synth.make_model(True, banks=banks(2, "concat", "dilate")),
    "dilate-n3-add": lambda: synth.make_model(True, banks=banks(3, "add", "dilate")),
    "bn-batch": lambda: bn_model(True),
    "bn-running": lambda: bn_model(False),
    "bn-batch-relu6": lambda: bn_model(True, relu6=True),
    "relu6-mres-n2-concat": lambda: bn_model(None, bk=banks(2, "concat", "mres"), relu6=True),
}
BATCH_STATS = {"bn-batch", "bn-batch-relu6"}

# case: (model, (nz, ny, nx), entry flags, entry velocity amplitudes).  'open': fluid on the x and z faces.  Where
# blocks straddle two entries (nb nz odd), an entry after the first is open and moving: a straddling block holds the
# last plane of one entry and the first of the next, and its sums must not all go to the first one's entry.
SCENES = {
    "default-quad-nb3": ("default", (9, 12, 32), ("geom", "open", "geom"), (0.0, 3.0, 8.0)),
    "default-box-nb2": ("default", (7, 8, 132), ("open", "geom"), (0.0, 3.0)),
    "mres-n2-concat-voxel-nb3": ("mres-n2-concat", (8, 12, 20), ("open", "geom", "geom"), (3.0, 8.0, 0.0)),
    "mres-n3-add-quad-nb2": ("mres-n3-add", (8, 12, 32), ("geom", "open"), (8.0, 3.0)),
    "dilate-n2-concat-voxel-nb2": ("dilate-n2-concat", (7, 10, 29), ("geom", "open"), (8.0, 3.0)),
    "dilate-n3-add-voxel-nb3": ("dilate-n3-add", (9, 11, 13), ("geom", "open", "geom"), (0.0, 3.0, 8.0)),
    "bn-batch-quad-nb3": ("bn-batch", (9, 12, 32), ("geom", "open", "geom"), (3.0, 8.0, 0.0)),
    "bn-running-box-nb2": ("bn-running", (7, 8, 132), ("geom", "open"), (3.0, 0.0)),
    "bn-batch-relu6-quad-nb2": ("bn-batch-relu6", (10, 12, 16), ("open", "geom"), (8.0, 3.0)),
    "relu6-mres-n2-concat-quad-nb3": ("relu6-mres-n2-concat", (8, 12, 16), ("geom", "open", "geom"), (0.0, 3.0, 8.0)),
}
MODES = ("tf32x3", "tf32")
CASES = [(s, m) for s in SCENES for m in MODES]
CASE_IDS = ["%s-%s" % c for c in CASES]


def kernel_kind(shape, nb):
    """'quad' or 'scalar': the fused step's kernels for this grid (quad_dims, tfl_fused.cu)."""
    nz, ny, nx = shape
    return "scalar" if quad_dims(nb, nz, ny, nx) is None else "quad"


def conv_kind(shape):
    return "box" if shape[2] > 128 else "zstream"


def test_scene_table_reaches_every_shape():
    """No GPU: every model in both modes, nb = 2 and 3, quad blocks straddling two entries, the per-voxel kernels, the
    box convolution, entries at rest and with open faces, dilated banks on grids 2 and 4 do not divide, small entries."""
    assert {s[0] for s in SCENES.values()} == set(MODELS)
    assert {len(s[2]) for s in SCENES.values()} == {2, 3}
    kinds = {kernel_kind(s[1], len(s[2])) for s in SCENES.values()}
    assert kinds == {"quad", "scalar"}
    straddle = [(sh, k) for _, sh, k, _ in SCENES.values() if (len(k) * sh[0]) % 2 == 1]
    assert {kernel_kind(sh, len(k)) for sh, k in straddle} == {"quad", "scalar"}
    assert all(any(k == "open" and a > 0 for k, a in zip(kinds_[1:], amps[1:]))
               for _, sh, kinds_, amps in SCENES.values() if (len(kinds_) * sh[0]) % 2 == 1)
    assert any(conv_kind(sh) == "box" for _, sh, _, _ in SCENES.values())
    assert sum(0.0 in amps for _, _, _, amps in SCENES.values()) >= len(SCENES) // 2
    for model, shape, kinds_, amps in SCENES.values():
        assert len(kinds_) == len(amps) and "open" in kinds_ and len(set(amps)) == len(amps)
        assert shape[0] * shape[1] * shape[2] <= 16 * 20 * 36
        if model.startswith("dilate"):
            assert any(n % 2 for n in shape), shape
        mnp = MODELS[model]()
        assert tc_covered(mnp), model
        assert all(takes_fused_path({"mode": m, "nb": len(kinds_), "pbc": False}) for m in MODES)


# ---------------------------------------------------------------------------------------------------------------
# Scenes
# ---------------------------------------------------------------------------------------------------------------
def entry_flags(kind, nz, ny, nx, seed):
    f = synth.make_flags(nx, ny, nz, True, nb=1, geometry=True, seed=seed)
    if kind == "open":
        f[:, :, :, 1:-1, 0] = synth.FLUID
        f[:, :, :, 1:-1, -1] = synth.FLUID
        f[:, :, 0, 1:-1, :] = synth.FLUID
        f[:, :, -1, 1:-1, :] = synth.FLUID
    return f


def make_scene(orc, shape, kinds, amps, seed=31):
    """Flags, U (amplitude 0: at rest), a small signed pDiv, density and plume BCs, each entry its own."""
    nz, ny, nx = shape
    flags = np.concatenate([entry_flags(k, nz, ny, nx, 7 + b) for b, k in enumerate(kinds)])
    U = np.concatenate([synth.make_smooth_velocity(flags[b:b + 1], True, amp=max(a, 1e-3), seed=seed + b) *
                        np.float32(a > 0) for b, a in enumerate(amps)])
    orc.setWallBcsForward(U, flags)
    batch = {"pDiv": (synth.make_density(flags, seed=seed + 7) - np.float32(0.5)) * np.float32(0.1), "UDiv": U,
             "flags": flags, "density": synth.make_density(flags, seed=seed + 8)}
    plume_bcs(batch, len(kinds))
    return {k: np.ascontiguousarray(v, np.float32) for k, v in batch.items()}


def gpu(batch):
    return {k: torch.from_numpy(np.ascontiguousarray(v).copy()).cuda() for k, v in batch.items()}


def host(batch):
    return {k: v.cpu().numpy() for k, v in batch.items()}


def entry(batch, b):
    return {k: np.ascontiguousarray(v[b:b + 1]) for k, v in batch.items()}


def oracle_tol(model, mode):
    """MODE_TOL, except for batch statistics in TF32: the statistics divide by the batch's standard deviation, which
    carries the 10-bit products' error into every voxel; on one H100 the relu6 model reached 3.4e-3 of p's max after
    two steps, inside the float64 bound (1) at every voxel.  3xTF32 stays within 2e-5."""
    return 1e-2 if model in BATCH_STATS and mode == "tf32" else MODE_TOL[mode]


def make_model(mnp, mode):
    gm = ProjectionModel.from_model(mnp)
    assert gm.get_mode() == "tf32x3"
    gm.set_mode(mode)
    return gm


# ---------------------------------------------------------------------------------------------------------------
# The batched fused step on every tensor-core model
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("scene,mode", CASES, ids=CASE_IDS)
def test_batched_fused_step(orc, scene, mode):
    from fluidnet_b200 import simulate, tfluids
    model, shape, kinds, amps = SCENES[scene]
    nb = len(kinds)
    mnp = MODELS[model]()
    gm = make_model(mnp, mode)
    fused = gpu(make_scene(orc, shape, kinds, amps))
    ctx = tfluids.context()
    ctx.trace_faults()
    worst = (0.0, 0.0)
    for step in range(3):
        ref = host(fused)
        state = {k: v.clone() for k, v in fused.items()}
        ops = {k: v.clone() for k, v in fused.items()}
        bound = projection_reference(state, MCONF, gm, mnp)
        oracle.simulate(orc, MCONF, ref, mnp, f64=True)
        simulate.simulate_fused(None, MCONF, fused, gm)
        simulate.simulate(None, MCONF, ops, gm)
        got, opg = host(fused), host(ops)
        what = "%s [%s] step %d" % (scene, mode, step)
        rp = check(what + " p vs float64", got["pDiv"], bound["p"], bound["Ep"])
        rU = check(what + " U vs float64", got["UDiv"], bound["U"], bound["EU"])
        worst = (max(worst[0], rp), max(worst[1], rU))
        for name, want in (("ops", opg), ("oracle", ref)):
            assert bits_equal(got["density"], want["density"]), "%s density vs %s: %s" % (
                what, name, describe_diff(got["density"], want["density"]))
        for k in ("UDiv", "pDiv"):
            close_per_entry(got[k], opg[k], OPS_TOL, "%s %s vs ops" % (what, k))
            assert same_zero_bits(got[k], opg[k]), "%s %s: zeros differ from the operator sequence" % (what, k)
            close_per_entry(got[k], ref[k], oracle_tol(model, mode), "%s %s vs oracle" % (what, k))
        if model in BATCH_STATS:
            other = {k: v.clone() for k, v in state.items()}
            other["UDiv"][1].mul_(2.0)
            simulate.simulate_fused(None, MCONF, other, gm)
            assert not torch.equal(other["pDiv"][0], fused["pDiv"][0]), "%s: entry 0 ignores entry 1" % what
        else:
            for b in range(nb):
                one = gpu(entry(host(state), b))
                simulate.simulate_fused(None, MCONF, one, gm)
                one = host(one)
                assert bits_equal(got["density"][b:b + 1], one["density"]), "%s entry %d density" % (what, b)
                for k in ("UDiv", "pDiv"):
                    close_per_entry(got[k][b:b + 1], one[k], OPS_TOL, "%s entry %d %s vs alone" % (what, b, k))
                    assert same_zero_bits(got[k][b:b + 1], one[k]), "%s entry %d %s zeros" % (what, b, k)
        assert ctx.trace_faults() == 0, what
    print("batched fused step %s [%s, %s kernels, %s conv, nb %d]: max err/E p %.3g U %.3g" % (
        scene, mode, kernel_kind(shape, nb), conv_kind(shape), nb, worst[0], worst[1]))


@pytest.mark.gpu
@pytest.mark.parametrize("scene", ["mres-n3-add-quad-nb2", "bn-batch-quad-nb3"])
def test_batched_graph_replays_equal_direct_steps(orc, scene):
    from fluidnet_b200 import simulate
    model, shape, kinds, amps = SCENES[scene]
    gm = make_model(MODELS[model](), "tf32x3")
    batch = make_scene(orc, shape, kinds, amps)
    stream = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(stream):
        direct, replayed = gpu(batch), gpu(batch)
        simulate.simulate_fused(None, MCONF, direct, gm)
        simulate.simulate_fused(None, MCONF, replayed, gm)
        graph = simulate.StepGraph(MCONF, replayed, gm)
        try:
            for step in range(4):
                if step >= 2:              # in-place changes between replays reach the captured tensors
                    for st in (direct, replayed):
                        st["density"][1].mul_(0.5)
                        st["UDiv"][0].mul_(-1.0 if step == 2 else 1.5)
                        st["pDiv"][-1].zero_()
                simulate.simulate_fused(None, MCONF, direct, gm)
                graph.launch()
                stream.synchronize()
                for k in ("pDiv", "UDiv", "density"):
                    a, b = direct[k].cpu().numpy(), replayed[k].cpu().numpy()
                    assert bits_equal(a, b), "%s replay %d %s: %s" % (scene, step, k, describe_diff(b, a))
        finally:
            graph.close()


def scene_kernels():
    """{case: (launch tally, {kernel: count})} of one fused step per case, under torch.profiler."""
    from fluidnet_b200 import simulate, tfluids
    from step_cases import tally_and_kernels
    orc = oracle.Oracle()
    out = {}
    for scene, mode in CASES:
        model, shape, kinds, amps = SCENES[scene]
        gm = make_model(MODELS[model](), mode)
        st = gpu(make_scene(orc, shape, kinds, amps))
        tally, kernels = tally_and_kernels(tfluids.context(), lambda: simulate.simulate_fused(None, MCONF, st, gm),
                                            attempts=6)
        out["%s-%s" % (scene, mode)] = (tally, dict(kernels))
    return out


@pytest.mark.gpu
def test_fused_kernels_ran():
    from step_cases import step_path
    seen = run_in_child("test_gpu_batch_models", "t.scene_kernels()")
    assert set(seen) == set(CASE_IDS)
    for (scene, mode), cid in zip(CASES, CASE_IDS):
        tally, kernels = seen[cid]
        _, shape, kinds, _ = SCENES[scene]
        path = step_path(kernels)
        print("batched fused step %s: %s kernels, %d launches" % (cid, path, tally))
        assert path == kernel_kind(shape, len(kinds)), (cid, path, sorted(kernels))
        assert tally == sum(kernels.values()), (cid, tally, kernels)


# ---------------------------------------------------------------------------------------------------------------
# calc_stats with batch statistics
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_calc_stats_batch_statistics_rows():
    """calc_stats at batch 3 with a batch-statistics model: the rows of a plain loop that steps the same batches of 3
    (the entries of a batch are coupled, so a loop over single frames would not do) with tfl_simulate_step, and
    reduces each state on the host."""
    from fluidnet_b200 import calc_stats, simulate, tfluids
    frames = calc_stats.synthetic_frames(7, 16, 5)
    gm = make_model(bn_model(True), "tf32x3")
    mconf = calc_stats.eval_mconf(None, "convnet")
    steps, size = 4, 3
    rows = calc_stats.run(frames, mconf, gm, steps, size, log=lambda *a: None)
    m = dict(mconf, is3D=True, normalizeInputThreshold=float(gm.threshold))
    want = []
    for first, part in calc_stats.group(frames, size):
        st = gpu({"pDiv": np.concatenate([f.p for f in part]), "UDiv": np.concatenate([f.U for f in part]),
                  "flags": np.concatenate([f.flags for f in part]), "density": np.concatenate([f.density for f in part])})
        div = torch.empty_like(st["pDiv"])
        vals = []
        for j in range(steps):
            if j:
                simulate.simulate_fused(None, m, st, gm)
            tfluids.velocityDivergenceForward(st["UDiv"], st["flags"], div)
            vals.append(monitor_reference.totals(monitor_reference.plane_partials(div.cpu().numpy(),
                                                                                 st["UDiv"].cpu().numpy())))
        for b, f in enumerate(part):
            for j in range(steps):
                dn, dm, um = vals[j][b]
                want.append((first + b, f.source, j + 1, dn, dm, um * m["dt"]))
    assert len(rows) == len(want) == 7 * steps
    for r, w in zip(rows, want):
        assert r[:3] == w[:3] and np.array_equal(np.array(r[3:]).view(np.uint64), np.array(w[3:]).view(np.uint64)), \
            (r, w)


# ---------------------------------------------------------------------------------------------------------------
# The launch grid's limits
# ---------------------------------------------------------------------------------------------------------------
MAX_GRID_YZ = 65535


def max_batch_planes(nz):
    """nb nz a grid may have: launch_dims / quad_dims / conv_launch / k_jacobi_iter4 give a block along gridDim.z two
    planes of a grid with nz > 1, one otherwise."""
    return 2 * MAX_GRID_YZ if nz > 1 else MAX_GRID_YZ


def max_rows(nz):
    """ny a grid may have: launch_dims gives a block along gridDim.y two rows of a grid with nz > 1, four otherwise."""
    return 2 * MAX_GRID_YZ if nz > 1 else 4 * MAX_GRID_YZ


def test_host_limit_matches_the_library():
    """No GPU: the limits restated here are the library's check_launch_grid (through tfl_debug_launch_grid_ok, host
    arithmetic only): at each limit accepted, one past it refused."""
    from fluidnet_b200 import _lib
    lib = C.CDLL(_lib.LIB_PATH)
    ok = lib.tfl_debug_launch_grid_ok
    ok.argtypes = [C.c_int32, C.c_int32, C.c_int32]
    for nz in (1, 2, 3, 5, 8, 300, 65535, 131070):
        nb = max_batch_planes(nz) // nz
        assert ok(nb, nz, 8) == 1, nz
        assert ok(nb + 1, nz, 8) == 0, nz
        assert ok(1, nz, max_rows(nz)) == 1 and ok(1, nz, max_rows(nz) + 1) == 0, nz
    assert ok(1, 131070, 8) == 1 and ok(1, 131071, 8) == 0          # one deep entry: the planes alone
    assert ok(65535, 1, 8) == 1 and ok(65536, 1, 8) == 0


def prototypes(orc, shape, is3d):
    """Four entries: geometry flags of their own, velocities of amplitude 3, 0 (at rest), 8 and 1, density, a small
    signed pDiv; no BCs."""
    nz, ny, nx = shape
    out = []
    for b, amp in enumerate((3.0, 0.0, 8.0, 1.0)):
        f = synth.make_flags(nx, ny, nz, is3d, nb=1, geometry=True, seed=40 + b)
        U = synth.make_smooth_velocity(f, is3d, amp=max(amp, 1e-3), seed=50 + b) * np.float32(amp > 0)
        orc.setWallBcsForward(U, f)
        out.append({"pDiv": (synth.make_density(f, seed=60 + b) - np.float32(0.5)) * np.float32(0.1), "UDiv": U,
                    "flags": f, "density": synth.make_density(f, seed=70 + b)})
    return [{k: np.ascontiguousarray(v, np.float32) for k, v in p.items()} for p in out]


def repeat(protos, nb):
    """The batch of nb entries, entry b a copy of prototype b % 4, built on the device."""
    out = {}
    for k in protos[0]:
        four = torch.from_numpy(np.concatenate([p[k] for p in protos])).cuda()
        out[k] = four.repeat((nb + 3) // 4, 1, 1, 1, 1)[:nb].contiguous()
    return out


def check_entries(got, want, what, tol=None):
    """Every entry b of the device tensor `got` against want[b % 4] (host): bit for bit, or within tol of its max."""
    nb = got.shape[0]
    for q in range(4):
        rows = got[q::4].cpu().numpy()
        w = want[q]
        if tol is None:
            same = (rows.view(np.uint32) == w.view(np.uint32)).reshape(rows.shape[0], -1).all(axis=1)
            assert same.all(), "%s: entries %s of prototype %d differ" % (what, (np.flatnonzero(~same) * 4 + q)[:8], q)
        else:
            err = np.abs(rows.astype(np.float64) - w.astype(np.float64)).reshape(rows.shape[0], -1).max(axis=1)
            scale = max(float(np.abs(w).max()), 1e-6)
            assert (err <= tol * scale).all(), "%s: prototype %d, worst err %g vs scale %g" % (what, q, err.max(), scale)
    assert nb > 4


def oracle_steps(orc, protos, mconf, mnp):
    """Each prototype stepped once by the oracle."""
    out = []
    for p in protos:
        one = {k: v.copy() for k, v in p.items()}
        oracle.simulate(orc, mconf, one, mnp)
        out.append(one)
    return out


def snapshot(st):
    return {k: v.clone() for k, v in st.items()}


def unchanged(st, before):
    return all(torch.equal(st[k].view(torch.int32), before[k].view(torch.int32)) for k in before)


LIMIT_GRIDS = {"2d-8x8": ((1, 8, 8), False), "3d-5x8x8": ((5, 8, 8), True)}


@pytest.mark.gpu
@pytest.mark.parametrize("grid", list(LIMIT_GRIDS))
def test_largest_batch_runs_and_one_more_is_refused(orc, grid):
    from fluidnet_b200 import monitor, simulate, tfluids
    from fluidnet_b200._lib import TflError
    shape, is3d = LIMIT_GRIDS[grid]
    nz = shape[0]
    nb = max_batch_planes(nz) // nz
    assert nb * nz == max_batch_planes(nz)
    protos = prototypes(orc, shape, is3d)
    mnp = synth.make_model(True)
    gm = ProjectionModel.from_model(mnp) if is3d else None
    jac = dict(JACOBI, is3D=is3d)
    ctx = tfluids.context()
    ctx.trace_faults()
    # the operator step (Jacobi) and, in 3-D, the fused convnet step
    for mconf, model in ([(jac, None)] + ([(MCONF, gm)] if is3d else [])):
        st = repeat(protos, nb)
        simulate.simulate_fused(None, mconf, st, model)
        want = oracle_steps(orc, protos, mconf, mnp if model else None)
        for k in ("density", "UDiv", "pDiv"):
            tol = None if model is None or k == "density" else MODE_TOL["tf32x3"]
            check_entries(st[k], [w[k] for w in want], "%s nb %d %s step %s" % (grid, nb, mconf["simMethod"], k), tol)
        del st
    # a Jacobi solve with pTol > 0 (k_sqdiff: one block row per entry)
    st = repeat(protos, nb)
    div = torch.from_numpy(np.concatenate([orc.velocityDivergenceForward(p["UDiv"], p["flags"]) for p in protos])
                           ).cuda().repeat((nb + 3) // 4, 1, 1, 1, 1)[:nb].contiguous()
    p_all = torch.zeros_like(st["pDiv"])
    res = tfluids.solveLinearSystemJacobi(p_all, st["flags"], div, is3d, 1e-9, 7)
    want, worst = [], 0.0
    for q, p in enumerate(protos):
        w = np.zeros_like(p["pDiv"])
        worst = max(worst, orc.solveLinearSystemJacobi(w, p["flags"], div[q:q + 1].cpu().numpy(), is3d, 1e-9, 7))
        want.append(w)
    check_entries(p_all, want, "%s jacobi pTol 1e-9" % grid)
    assert abs(res - worst) <= 1e-5 * worst, (res, worst)
    # the monitor
    with monitor.StepMonitor(None, st, 2) as mon:
        mon.record(st)
        _, vals = mon.take()
    for q, p in enumerate(protos):
        rec = monitor_reference.record(orc, p["UDiv"], p["flags"])
        assert np.array_equal(vals[q::4], np.broadcast_to(rec, vals[q::4].shape)), (grid, q)
    assert ctx.trace_faults() == 0
    del st, div, p_all
    # one entry more: refused by name before anything runs, the state untouched
    big = repeat(protos, nb + 1)
    before = snapshot(big)
    limit = "at most %d" % (max_batch_planes(nz) if is3d else MAX_GRID_YZ)
    calls = [lambda: simulate.simulate_fused(None, jac, big, None),
             lambda: tfluids.solveLinearSystemJacobi(big["pDiv"], big["flags"], big["density"], is3d, 1e-9, 7)]
    if is3d:
        calls.append(lambda: simulate.simulate_fused(None, MCONF, big, gm))

    def monitored():
        with monitor.StepMonitor(None, big, 2) as mon:
            mon.record(big)
    calls.append(monitored)
    for call in calls:
        n0 = ctx.launch_count()
        with pytest.raises(TflError, match=limit):
            call()
        torch.cuda.synchronize()
        assert ctx.launch_count() == n0
        assert unchanged(big, before)
    del big, before
    # the context still steps a valid batch
    st = repeat(protos, 8)
    simulate.simulate_fused(None, jac, st, None)
    want = oracle_steps(orc, protos, jac, None)
    for k in ("density", "UDiv", "pDiv"):
        check_entries(st[k], [w[k] for w in want], "%s after the refusals: %s" % (grid, k))
    assert ctx.trace_faults() == 0
