"""Batches of independent 3-D scenes on the fast path: the advection tiles over the batch axis, the fused step at
nb > 1, and calc_stats' per-scene table.

  * Tiles: each entry of a batch whose entries differ (flags sphere + slab / open / exotic, traces of 0.2, 0.8 and
    2.5 cells) equals the oracle on that entry alone, bit for bit, under every tile mode, with no trace fault; modes 1
    and 2 save exactly one launch per field over mode 0 whatever nb is.
  * Entry independence: each entry of a batched step equals the same scene stepped alone at nb = 1 -- Jacobi bit for
    bit over 20 steps, convnet one step at a time (density bit for bit, U and p within test_gpu_step_paths' 1e-6 of
    the entry's max with the same exact zeros, and within MODE_TOL of the oracle).
  * The batched step graph and tfl_host_sim_step equal the direct batched step; the fused step's launch tally does
    not depend on nb and matches what torch.profiler sees; the monitor's records and a recorded frame of one entry
    equal that entry stepped alone; calc_stats' rows equal a plain loop."""
import ctypes as C
import json
import os
import subprocess
import sys
from collections import Counter

import numpy as np
import pytest
import torch

import edge_cases
import monitor_reference
import oracle
from cases import bits_equal, describe_diff
from fluidnet_b200 import synth
from step_cases import MODE_TOL, OPS_TOL, close_per_entry, fill, plane_of, plume_bcs, run, same_zero_bits, set_tile_mode

pytestmark = pytest.mark.gpu

DT, STRENGTH = edge_cases.DT, edge_cases.STRENGTH
KINDS = ("geom", "open", "exotic")
TRACES = (0.2, 0.8, 2.5)


def entry_flags(kind, nz, ny, nx, seed):
    f = synth.make_flags(nx, ny, nz, True, nb=1, geometry=kind != "empty", exotic=kind == "exotic", seed=seed)
    if kind == "open":           # fluid on the x and z faces: a box crossing into the next entry changes bits
        f[:, :, :, 1:-1, 0] = synth.FLUID
        f[:, :, :, 1:-1, -1] = synth.FLUID
        f[:, :, 0, 1:-1, :] = synth.FLUID
        f[:, :, -1, 1:-1, :] = synth.FLUID
    return f


def batch_fields(orc, shape, kinds, traces, seed=11):
    """flags, U (wall BCs applied), a scalar: one entry per (kind, trace), each with its own seed."""
    nz, ny, nx = shape
    fl, U, s = [], [], []
    for b, (kind, trace) in enumerate(zip(kinds, traces)):
        f = entry_flags(kind, nz, ny, nx, seed + b)
        u = synth.make_smooth_velocity(f, True, amp=trace / DT, seed=seed + 10 * b)
        orc.setWallBcsForward(u, f)
        fl.append(f)
        U.append(u)
        s.append(synth.make_density(f, seed=seed + 10 * b + 1))
    cat = lambda a: np.ascontiguousarray(np.concatenate(a))          # noqa: E731
    return cat(fl), cat(U), cat(s)


TILE_CASES = {
    "nb2-geom-open-z10": ((10, 12, 32), ("geom", "open"), (0.2, 2.5)),
    "nb3-all-z9-x36": ((9, 11, 36), KINDS, TRACES),
    "nb3-all-z16": ((16, 8, 32), ("open", "exotic", "geom"), (0.8, 0.2, 2.5)),
}


@pytest.mark.parametrize("name", list(TILE_CASES))
def test_tiles_per_entry_equal_the_oracle(orc, name):
    from fluidnet_b200 import tfluids
    shape, kinds, traces = TILE_CASES[name]
    fl, U, s = batch_fields(orc, shape, kinds, traces)
    nb = fl.shape[0]
    pl = plane_of(fl)
    want_s = {o: np.concatenate([orc.advectScalar(DT, s[b:b + 1], U[b:b + 1], fl[b:b + 1], "maccormackOurs", o,
                                                 STRENGTH) for b in range(nb)]) for o in (False, True)}
    want_u = np.concatenate([orc.advectVel(DT, U[b:b + 1], fl[b:b + 1], "maccormackOurs", STRENGTH) for b in range(nb)])
    counts = {}
    try:
        for mode in (None, 0, 1, 2):
            set_tile_mode(mode)
            tag = "%s tile %s" % (name, mode)
            for o in (False, True):
                (_, _, _, got), _, n = run("advectScalar " + tag, pl, lambda ts, tu, tf, d: tfluids.advectScalar(
                    DT, ts, tu, tf, "maccormackOurs", d, o, STRENGTH), s, U, fl, fill(s.shape))
                for b in range(nb):
                    assert bits_equal(got[b], want_s[o][b]), "%s outside %s entry %d: %s" % (
                        tag, o, b, describe_diff(got[b], want_s[o][b]))
                counts[("s", o, mode)] = n
            (_, _, got), _, n = run("advectVel " + tag, pl, lambda tu, tf, d: tfluids.advectVel(
                DT, tu, tf, "maccormackOurs", d, STRENGTH), U, fl, fill(U.shape))
            for b in range(nb):
                assert bits_equal(got[b], want_u[b]), "%s advectVel entry %d: %s" % (tag, b, describe_diff(got[b],
                                                                                                       want_u[b]))
            counts[("u", None, mode)] = n
    finally:
        set_tile_mode(None)
    for mode in (1, 2):
        for key in (("s", False), ("s", True), ("u", None)):
            assert counts[key + (mode,)] == counts[key + (0,)] - 1, (name, key, mode, counts)


# ---------------------------------------------------------------------------------------------------------------
# Entry independence: the batched step against each entry stepped alone
# ---------------------------------------------------------------------------------------------------------------
def step_batch(orc, shape, nb, amps, seed=21, kind="geom"):
    """A plume state per entry: geometry flags (kind 'open': fluid also on the x and z faces, so that the first and
    last planes of an entry carry velocity into the input scale's sums), its own velocity amplitude (0: at rest),
    density and plume BCs of its own radius (plume_bcs)."""
    nz, ny, nx = shape
    flags = np.concatenate([entry_flags(kind, nz, ny, nx, 7) for _ in range(nb)])
    U = np.concatenate([synth.make_smooth_velocity(flags[b:b + 1], True, amp=max(a, 1e-3), seed=seed + b) *
                        np.float32(a > 0) for b, a in enumerate(amps)])
    orc.setWallBcsForward(U, flags)
    batch = {"pDiv": (synth.make_density(flags, seed=seed + 7) - np.float32(0.5)) * np.float32(0.1), "UDiv": U,
             "flags": flags, "density": synth.make_density(flags, seed=seed + 8)}
    plume_bcs(batch, nb)
    return {k: np.ascontiguousarray(v, np.float32) for k, v in batch.items()}


def entry(batch, b):
    return {k: np.ascontiguousarray(v[b:b + 1]) for k, v in batch.items()}


def gpu(batch):
    return {k: torch.from_numpy(v.copy()).cuda() for k, v in batch.items()}


def host(batch):
    return {k: v.cpu().numpy() for k, v in batch.items()}


JACOBI = oracle.default_mconf(dt=0.1, maccormackStrength=0.6, buoyancyScale=0.5, vorticityConfinementAmp=3.0,
                              simMethod="jacobi", maxIter=34)
CONVNET = oracle.default_mconf(dt=0.1, maccormackStrength=0.6, buoyancyScale=0.5, vorticityConfinementAmp=3.0,
                               simMethod="convnet")


def test_jacobi_entries_equal_alone(orc):
    from fluidnet_b200 import simulate, tfluids
    shape, amps = (9, 12, 32), (3.0, 0.0, 8.0)
    batch = step_batch(orc, shape, 3, amps)
    together = gpu(batch)
    alone = [gpu(entry(batch, b)) for b in range(3)]
    ctx = tfluids.context()
    ctx.trace_faults()
    for step in range(20):
        simulate.simulate_fused(None, JACOBI, together, None)
        for a in alone:
            simulate.simulate_fused(None, JACOBI, a, None)
        got = host(together)
        for b in range(3):
            one = host(alone[b])
            for k in ("pDiv", "UDiv", "density"):
                assert bits_equal(got[k][b:b + 1], one[k]), "step %d entry %d %s: %s" % (
                    step, b, k, describe_diff(got[k][b:b + 1], one[k]))
    assert ctx.trace_faults() == 0


# (shape, per-entry velocity amplitudes, flags): quad kernels with nb * nz odd (a block straddles two entries); the
# per-voxel kernels (nx % 4 != 0, no tile) with an odd nz (blocks of two planes straddle too); partial x and y quad
# blocks; an entry at rest.  Where blocks straddle, the z faces are fluid: the straddling blocks hold the last plane of
# one entry and the first of the next, and with solid faces both would add nothing to the sums.
STEP_CASES = {
    "quad-odd-nbnz-open": ((9, 12, 32), (3.0, 0.0, 8.0), "open"),
    "voxel-nx18-open": ((7, 10, 18), (3.0, 8.0), "open"),
    "quad-partial-xy": ((6, 11, 132), (0.0, 3.0), "geom"),
}


@pytest.mark.parametrize("mode", ["tf32x3", "tf32"])
@pytest.mark.parametrize("name", list(STEP_CASES))
def test_convnet_entries_equal_alone(orc, name, mode):
    from fluidnet_b200 import simulate, tfluids
    from fluidnet_b200.model import ProjectionModel
    shape, amps, kind = STEP_CASES[name]
    nb = len(amps)
    batch = step_batch(orc, shape, nb, amps, kind=kind)
    mnp = synth.make_model(True)
    gm = ProjectionModel.from_model(mnp)
    gm.set_mode(mode)
    together = gpu(batch)
    ctx = tfluids.context()
    ctx.trace_faults()
    for step in range(3):
        ref = host(together)
        alone = [gpu(entry(ref, b)) for b in range(nb)]
        simulate.simulate_fused(None, CONVNET, together, gm)
        for a in alone:
            simulate.simulate_fused(None, CONVNET, a, gm)
        oracle.simulate(orc, CONVNET, ref, mnp)
        got = host(together)
        what = "%s %s step %d" % (name, mode, step)
        for b in range(nb):
            one = host(alone[b])
            assert bits_equal(got["density"][b:b + 1], one["density"]), "%s entry %d density: %s" % (
                what, b, describe_diff(got["density"][b:b + 1], one["density"]))
            for k in ("UDiv", "pDiv"):
                close_per_entry(got[k][b:b + 1], one[k], OPS_TOL, "%s entry %d %s vs alone" % (what, b, k))
                assert same_zero_bits(got[k][b:b + 1], one[k]), "%s entry %d %s zeros" % (what, b, k)
        assert bits_equal(got["density"], ref["density"]), "%s density vs oracle" % what
        for k in ("UDiv", "pDiv"):
            close_per_entry(got[k], ref[k], MODE_TOL[mode], "%s %s vs oracle" % (what, k))
    assert ctx.trace_faults() == 0


def test_large_batches(orc):
    """nb = 100 tiny scenes through the fused step (z range 5: blocks straddle entries) and nb = 300 through a Jacobi
    solve with a tolerance (the per-entry residual sums): every per-entry buffer grows with nb."""
    from fluidnet_b200 import simulate, tfluids
    from fluidnet_b200.model import ProjectionModel
    four = step_batch(orc, (5, 8, 8), 4, (3.0, 0.0, 8.0, 1.0), kind="open")
    many = {k: np.ascontiguousarray(np.concatenate([v[b % 4:b % 4 + 1] for b in range(100)])) for k, v in four.items()}
    gm = ProjectionModel.from_model(synth.make_model(True))
    gm.set_mode("tf32x3")
    together = gpu(many)
    alone = [gpu(entry(four, b)) for b in range(4)]
    for step in range(2):
        simulate.simulate_fused(None, CONVNET, together, gm)
        for a in alone:
            simulate.simulate_fused(None, CONVNET, a, gm)
        got = host(together)
        for b in range(100):
            one = host(alone[b % 4])
            assert bits_equal(got["density"][b:b + 1], one["density"]), "step %d entry %d density" % (step, b)
            for k in ("UDiv", "pDiv"):
                close_per_entry(got[k][b:b + 1], one[k], OPS_TOL, "step %d entry %d %s" % (step, b, k))
    # Jacobi with pTol > 0: the residual is the largest of the per-entry norms
    flags = np.ascontiguousarray(np.concatenate([four["flags"][b % 4:b % 4 + 1] for b in range(300)]))
    div = np.ascontiguousarray((synth.make_density(flags, seed=3) - np.float32(0.5)), np.float32)
    p_all = torch.zeros(flags.shape, device="cuda")
    res_all = tfluids.solveLinearSystemJacobi(p_all, torch.from_numpy(flags).cuda(), torch.from_numpy(div).cuda(),
                                              True, 1e-9, 7)
    worst = 0.0
    for b in range(300):
        p1 = torch.zeros(flags[b:b + 1].shape, device="cuda")
        r1 = tfluids.solveLinearSystemJacobi(p1, torch.from_numpy(flags[b:b + 1].copy()).cuda(),
                                             torch.from_numpy(div[b:b + 1].copy()).cuda(), True, 1e-9, 7)
        worst = max(worst, r1)
        assert bits_equal(p_all[b:b + 1].cpu().numpy(), p1.cpu().numpy()), "jacobi entry %d" % b
    assert abs(res_all - worst) <= 1e-6 * worst, (res_all, worst)    # the same fp64 sums, each rounded to float


# ---------------------------------------------------------------------------------------------------------------
# Graph and host-buffer paths, launches
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("method", ["convnet", "jacobi"])
def test_batched_graph_replays_equal_direct_steps(orc, method):
    from fluidnet_b200 import simulate
    from fluidnet_b200.model import ProjectionModel
    mconf = CONVNET if method == "convnet" else JACOBI
    batch = step_batch(orc, (8, 12, 32), 3, (3.0, 0.0, 8.0))
    gm = ProjectionModel.from_model(synth.make_model(True)) if method == "convnet" else None
    if gm is not None:
        gm.set_mode("tf32x3")
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        direct, replayed = gpu(batch), gpu(batch)
        simulate.simulate_fused(None, mconf, direct, gm)
        simulate.simulate_fused(None, mconf, replayed, gm)
        graph = simulate.StepGraph(mconf, replayed, gm)
        try:
            for step in range(5):
                if step == 2:              # in-place changes between replays reach the captured tensors
                    for st in (direct, replayed):
                        st["density"][1].mul_(0.5)
                        st["UDiv"][0].mul_(-1.0)
                simulate.simulate_fused(None, mconf, direct, gm)
                graph.launch()
                stream.synchronize()
                for k in ("pDiv", "UDiv", "density"):
                    a, b = direct[k].cpu().numpy(), replayed[k].cpu().numpy()
                    assert bits_equal(a, b), "%s step %d %s: %s" % (method, step, k, describe_diff(b, a))
        finally:
            graph.close()


def test_host_buffer_step_at_nb3(orc):
    from fluidnet_b200 import simulate, tfluids
    from fluidnet_b200.model import ProjectionModel
    shape = (9, 12, 32)
    batch = step_batch(orc, shape, 3, (3.0, 0.0, 8.0))
    gm = ProjectionModel.from_model(synth.make_model(True))
    gm.set_mode("tf32x3")
    dev = gpu(batch)
    ctx = tfluids.context()
    lib = ctx.lib
    hs = C.c_void_p()
    keep = [np.ascontiguousarray(batch[k]) for k in ("flags", "UBC", "UBCInvMask", "densityBC", "densityBCInvMask")]
    nz, ny, nx = shape
    ctx.check(lib.tfl_host_sim_create(ctx.h, 3, nz, ny, nx, 1, *[a.ctypes.data for a in keep], C.byref(hs)))
    hp = torch.from_numpy(batch["pDiv"].copy()).pin_memory()
    hU = torch.from_numpy(batch["UDiv"].copy()).pin_memory()
    hd = torch.from_numpy(batch["density"].copy()).pin_memory()
    mc = simulate.make_mconf(CONVNET)
    mc.normalize_input_threshold = float(gm.threshold)
    try:
        for step in range(2):
            simulate.simulate_fused(None, CONVNET, dev, gm)
            ctx.check(lib.tfl_host_sim_step(ctx.h, hs, hp.data_ptr(), hU.data_ptr(), hd.data_ptr(), C.byref(mc),
                                            gm.h))
            assert bits_equal(hd.numpy(), dev["density"].cpu().numpy()), "step %d density" % step
            for k, h in (("UDiv", hU), ("pDiv", hp)):
                close_per_entry(h.numpy(), dev[k].cpu().numpy(), OPS_TOL, "step %d %s" % (step, k))
    finally:
        lib.tfl_host_sim_destroy(ctx.h, hs)


def _profiled(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return Counter(ev.name for ev in prof.events()
                   if ev.device_type == torch.autograd.DeviceType.CUDA and not ev.name.startswith(("Memcpy", "Memset")))


def _tally_and_kernels(ctx, call, attempts=3):
    """(tally `call` added, kernels the profiler saw), the capture bracketed by two marker kernels as in
    test_gpu_launch_tally.py: a capture that lost a marker is taken again."""
    call()
    torch.cuda.synchronize()
    buf = torch.zeros(1, device="cuda")
    mark = lambda: buf.add_(1.0)                # noqa: E731
    for _ in range(attempts):
        marks = _profiled(lambda: (mark(), mark()))
        if sum(marks.values()) != 2:
            continue
        before = ctx.launch_count()
        seen = _profiled(lambda: (mark(), call(), mark()))
        tally = ctx.launch_count() - before
        if all(seen[k] >= n for k, n in marks.items()):
            return tally, seen - marks
    raise AssertionError("the profiler lost its marker kernels in %d captures" % attempts)


def launch_census(nb):
    """{n: (tally, {kernel: count})} of one fused step at n = 1 and n = nb, under torch.profiler in this process."""
    from fluidnet_b200 import simulate, tfluids
    from fluidnet_b200.model import ProjectionModel
    orc = oracle.Oracle()
    gm = ProjectionModel.from_model(synth.make_model(True))
    gm.set_mode("tf32x3")
    ctx = tfluids.context()
    out = {}
    for n in (1, nb):
        st = gpu(step_batch(orc, (16, 16, 32), n, (3.0,) * n))
        tally, kernels = _tally_and_kernels(ctx, lambda: simulate.simulate_fused(None, CONVNET, st, gm))
        out[n] = (tally, dict(kernels))
    return out


@pytest.mark.parametrize("nb", [2, 5])
def test_fused_step_launches_do_not_depend_on_nb(nb):
    # The profiler runs in a child process: on one H100 run, a profiler session opened in the test process left every
    # capture of test_gpu_launch_tally.py, later in the same process, without a kernel event.
    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ)
    env["PYTHONPATH"] = os.pathsep.join(p for p in (here, os.path.dirname(here), env.get("PYTHONPATH")) if p)
    code = "import json, test_gpu_batch as t; print(json.dumps(t.launch_census(%d)))" % nb
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env, timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    census = {int(k): v for k, v in json.loads(r.stdout.strip().splitlines()[-1]).items()}
    for n, (tally, kernels) in census.items():
        assert tally == sum(kernels.values()), (n, tally, kernels)
    kernels = census[nb][1]
    assert any("k_advect_vel_tile" in k for k in kernels) and any("k_post_advect4" in k for k in kernels), kernels
    assert census[1][0] == census[nb][0], census


# ---------------------------------------------------------------------------------------------------------------
# Monitor and recorder on entries of a batch
# ---------------------------------------------------------------------------------------------------------------
def test_monitor_and_frames_of_batched_entries(orc):
    from fluidnet_b200 import monitor, record, simulate
    shape = (9, 12, 32)
    batch = step_batch(orc, shape, 3, (3.0, 0.0, 8.0))
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        together = gpu(batch)
        alone = [gpu(entry(batch, b)) for b in range(3)]
        simulate.simulate_fused(None, JACOBI, together, None)
        for a in alone:
            simulate.simulate_fused(None, JACOBI, a, None)
        with monitor.StepMonitor(None, together, 4) as mon:
            mon.record(together)
            _, vals = mon.take()
        for b in range(3):
            with monitor.StepMonitor(None, alone[b], 4) as mon:
                mon.record(alone[b])
                _, one = mon.take()
            assert np.array_equal(vals[b].view(np.uint64), one[0].view(np.uint64)), (b, vals[b], one[0])
            want = monitor_reference.record(orc, alone[b]["UDiv"].cpu().numpy(), alone[b]["flags"].cpu().numpy())
            assert np.array_equal(one, want), (b, one, want)
            rec = record.FrameRecorder(shape)
            try:
                rec.capture(together["density"][b:b + 1])
                _, frame = rec.take(True)
                got = np.array(frame).transpose(2, 1, 0)
                rec.release()
            finally:
                rec.close()
            assert bits_equal(got, alone[b]["density"].cpu().numpy()[0, 0]), "entry %d frame" % b


# ---------------------------------------------------------------------------------------------------------------
# calc_stats
# ---------------------------------------------------------------------------------------------------------------
def _plain_loop(frames, mconf, steps, model=None):
    """Each frame alone: simulate (operator by operator), velocityDivergenceForward, the monitor's reduction restated
    on the host -> rows as calc_stats writes them."""
    from fluidnet_b200 import simulate, tfluids
    rows = []
    for i, f in enumerate(frames):
        st = {"pDiv": torch.from_numpy(f.p.copy()).cuda(), "UDiv": torch.from_numpy(f.U.copy()).cuda(),
              "flags": torch.from_numpy(f.flags.copy()).cuda(), "density": torch.from_numpy(f.density.copy()).cuda()}
        m = dict(mconf, is3D=f.is3d)
        if model is not None:
            m["normalizeInputThreshold"] = float(model.threshold)
        div = torch.empty_like(st["pDiv"])
        for j in range(steps):
            if j:
                simulate.simulate(None, m, st, model)
            tfluids.velocityDivergenceForward(st["UDiv"], st["flags"], div)
            d, U = div.cpu().numpy(), st["UDiv"].cpu().numpy()
            dn, dm, um = monitor_reference.totals(monitor_reference.plane_partials(d, U))[0]
            rows.append((i, f.source, j + 1, dn, dm, um * m["dt"]))
    return rows


def test_calc_stats_rows_equal_a_plain_loop(tmp_path):
    from fluidnet_b200 import calc_stats, formats
    frames = calc_stats.synthetic_frames(7, 16, 3)
    paths = []
    for i, f in enumerate(frames):
        paths.append(str(tmp_path / ("frame%02d.bin" % i)))
        formats.save_manta_file(paths[-1], f.p, f.U, f.flags, f.density)
    loaded = calc_stats.load_frames(paths)
    mconf = calc_stats.eval_mconf(None, "jacobi")
    steps = 6
    rows3 = calc_stats.run(loaded, mconf, None, steps, 3, log=lambda *a: None)
    rows1 = calc_stats.run(loaded, mconf, None, steps, 1, log=lambda *a: None)
    want = _plain_loop(loaded, mconf, steps)
    assert len(rows3) == 7 * steps
    for got in (rows3, rows1):
        for r, w in zip(got, want):
            assert r[:3] == w[:3] and np.array_equal(np.array(r[3:]).view(np.uint64), np.array(w[3:]).view(np.uint64)), \
                (r, w)
    out = str(tmp_path / "stats.csv")
    calc_stats.write_csv(out, rows3)
    assert calc_stats.read_csv(out) == [tuple(r) for r in rows3]


def test_calc_stats_2d_frames():
    """2-D frames run on the operator path, with the same step graph and monitor."""
    from fluidnet_b200 import calc_stats
    frames = calc_stats.synthetic_frames(5, 16, 4, is3d=False)
    mconf = calc_stats.eval_mconf(None, "jacobi")
    rows = calc_stats.run(frames, mconf, None, 5, 2, log=lambda *a: None)
    want = _plain_loop(frames, mconf, 5)
    assert len(rows) == 25
    for r, w in zip(rows, want):
        assert r[:3] == w[:3] and np.array_equal(np.array(r[3:]).view(np.uint64), np.array(w[3:]).view(np.uint64)), \
            (r, w)


def test_calc_stats_convnet_batches(tmp_path):
    """The convnet table through the fused step: the start frame's row is exact, later rows stay close to the plain
    operator loop (the conv stack and the input scale's double atomics)."""
    from fluidnet_b200 import calc_stats
    from fluidnet_b200.model import ProjectionModel
    frames = calc_stats.synthetic_frames(5, 16, 9)
    gm = ProjectionModel.from_model(synth.make_model(True))
    gm.set_mode("tf32x3")
    mconf = calc_stats.eval_mconf(None, "convnet")
    rows = calc_stats.run(frames, mconf, gm, 4, 2, log=lambda *a: None)
    want = _plain_loop(frames, mconf, 4, gm)
    for r, w in zip(rows, want):
        assert r[:3] == w[:3]
        if r[2] == 1:
            assert r[3:] == w[3:], (r, w)
        else:
            assert np.allclose(r[3:], w[3:], rtol=1e-3, atol=1e-5), (r, w)
