"""tfl_launch_count against the kernels that really ran: each case runs once to warm up, then under torch.profiler
with CUDA activities, and the number of kernel events (memcpy and memset left out) must equal what the call added to
the context's tally.  The cases walk the projection network's drivers: tfl_cnn_project on the fp32 path (plain loop
and graph executor) and on the tensor cores (single bank, banked 'mres' and 'dilate' stacks, batch statistics, the
pressure skip), the fused tfl_simulate_step, and a single-rank tfl_slab_sim_step with a banked model."""
import warnings
from collections import Counter

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def banks(num, agg, typ="mres"):
    return {"num": num, "split_stage": 1, "join_stage": 3, "aggregate": agg, "type": typ}


def _model(mnp, mode):
    from fluidnet_b200 import model as fmodel
    kw = {k: mnp[k] for k in ("pool", "up", "poolType", "nonlinType", "banks", "batchNorm") if k in mnp}
    kw.update(mnp.get("inputs") or {})
    gm = fmodel.ProjectionModel(mnp["layers"], mnp["is3D"], **kw)
    gm.set_mode(mode)
    return gm


def _fields(nz, ny, nx, is3d=True):
    import oracle
    from fluidnet_b200 import synth
    flags = synth.make_flags(nx, ny, nz, is3d, nb=1, geometry=True)
    U = synth.make_smooth_velocity(flags, is3d, amp=3.0)
    oracle.Oracle().setWallBcsForward(U, flags)
    p = (np.random.RandomState(5).rand(*flags.shape).astype(np.float32) - 0.5)
    return {"pDiv": p, "UDiv": U, "flags": flags, "density": synth.make_density(flags)}


def _profiled_kernels(fn):
    """Counter of the kernels (memcpy and memset left out) the profiler saw while fn ran."""
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return Counter(ev.name for ev in prof.events()
                   if ev.device_type == torch.autograd.DeviceType.CUDA
                   and not ev.name.startswith(("Memcpy", "Memset")))


def _tally_and_kernels(ctx, call, attempts=3):
    """(what `call` added to ctx's launch tally, Counter of the kernels the profiler saw it run).

    The profiler can lose a whole capture: on one H100 run it reported no kernel at all for a step that had enqueued
    20.  So every capture brackets the call with two marker kernels of known names (one torch add each), and a capture
    that misses a marker proves nothing about the call: it is taken again, and after `attempts` such captures the
    test fails.  The markers are removed from the count exactly; everything else the capture saw is the call's."""
    call()
    torch.cuda.synchronize()
    buf = torch.zeros(1, device="cuda")
    mark = lambda: buf.add_(1.0)
    lost = 0
    for _ in range(attempts):
        marks = _profiled_kernels(lambda: (mark(), mark()))
        if sum(marks.values()) != 2:
            lost += 1
            continue
        before = ctx.launch_count()
        seen = _profiled_kernels(lambda: (mark(), call(), mark()))
        tally = ctx.launch_count() - before
        if all(seen[k] >= n for k, n in marks.items()):
            if lost:
                warnings.warn("the profiler lost %d capture(s) before this one" % lost)
            return tally, seen - marks
        lost += 1
    raise AssertionError("the profiler lost its marker kernels in %d captures out of %d" % (lost, attempts))


def _check(ctx, call, what):
    tally, kernels = _tally_and_kernels(ctx, call)
    assert tally == sum(kernels.values()), (what, "tallied %d, ran %d" % (tally, sum(kernels.values())), dict(kernels))


# (id, synth.make_model keywords, mode, grid nz ny nx)
PROJECT = [
    ("default-fp32", {}, "fp32", (16, 16, 16)),
    ("default-tf32", {}, "tf32", (16, 16, 16)),
    ("default-tf32x3", {}, "tf32x3", (16, 16, 16)),
    ("mres3-concat-tf32x3", {"banks": banks(3, "concat")}, "tf32x3", (16, 16, 16)),
    ("mres3-concat-fp32", {"banks": banks(3, "concat")}, "fp32", (16, 16, 16)),
    ("mres3-add-tf32x3", {"banks": banks(3, "add")}, "tf32x3", (16, 16, 16)),
    ("mres3-add-fp32", {"banks": banks(3, "add")}, "fp32", (16, 16, 16)),
    # 2 does not divide 15: the short phases of the dilated bank are re-zeroed
    ("dilate2-concat-tf32x3", {"banks": banks(2, "concat", "dilate")}, "tf32x3", (15, 16, 15)),
    ("dilate2-add-fp32", {"banks": banks(2, "add", "dilate")}, "fp32", (15, 16, 15)),
    ("bn-batch-tf32x3", {"batch_norm": {"train": True}}, "tf32x3", (16, 16, 16)),
    ("bn-batch-fp32", {"batch_norm": {"train": True}}, "fp32", (16, 16, 16)),
    ("skip-tf32x3", {"inputs": {"addPressureSkip": True}}, "tf32x3", (16, 16, 16)),
    ("skip-div-scale-fp32", {"inputs": {"addPressureSkip": True, "normalizeInputChan": "div"}}, "fp32", (16, 16, 16)),
    ("tog-fp32", {"model_type": "tog"}, "fp32", (16, 16, 16)),
]


@pytest.mark.parametrize("case", PROJECT, ids=[c[0] for c in PROJECT])
def test_cnn_project_tallies_the_kernels_it_runs(case):
    from fluidnet_b200 import synth
    name, kw, mode, (nz, ny, nx) = case
    gm = _model(synth.make_model(True, **kw), mode)
    f = {k: torch.from_numpy(v).cuda() for k, v in _fields(nz, ny, nx).items()}
    out = (torch.empty_like(f["pDiv"]), torch.empty_like(f["UDiv"]))
    _check(gm.ctx, lambda: gm.forward((f["pDiv"], f["UDiv"], f["flags"]), out=out), name)


def _step_problem(n, bk):
    import oracle
    from fluidnet_b200 import synth
    batch = _fields(n, n, n)
    batch["pDiv"] = np.zeros_like(batch["flags"])
    oracle.create_plume_bcs(batch, [1.0], n / 128.0 * 4, 0.15)
    mconf = oracle.default_mconf(dt=0.1, maccormackStrength=0.6, buoyancyScale=2.0 * n / 128,
                                 vorticityConfinementAmp=3.0, simMethod="convnet")
    return batch, mconf, synth.make_model(True, banks=bk)


@pytest.mark.parametrize("bk", [None, banks(2, "concat")], ids=["default", "mres2-concat"])
def test_fused_step_tallies_the_kernels_it_runs(bk):
    from fluidnet_b200 import simulate
    batch, mconf, mnp = _step_problem(32, bk)
    gm = _model(mnp, "tf32x3")
    gb = {k: torch.from_numpy(v).cuda() for k, v in batch.items()}
    _check(gm.ctx, lambda: simulate.simulate_fused(None, mconf, gb, gm), "tfl_simulate_step")


def test_single_rank_slab_step_tallies_the_kernels_it_runs():
    from fluidnet_b200.slab import NativeSlabSimulator
    bk = banks(2, "concat")
    del bk["type"]
    batch, mconf, mnp = _step_problem(32, bk)
    tb = {k: torch.from_numpy(v) for k, v in batch.items()}
    sim = NativeSlabSimulator(tb, mconf, mnp["layers"], torch.device("cuda", 0), rank=0, world=1, banks=bk)
    try:
        _check(sim.ctx, sim.step, "tfl_slab_sim_step")
    finally:
        sim.close()
