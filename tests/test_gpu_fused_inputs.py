"""The fused step (tfl_simulate_step's fused pipeline) with every input block of the projection network on the tensor
cores: inputChannels with UDiv, normalizeInputFunc 'norm', normalizeInputChan 'pDiv' and 'div', the pressure skip and
normalizeInput off.

  (1) Per voxel against float64: one step of a plume problem with a signed pDiv, for each block of INPUTS in 3xTF32
      and TF32 at nb = 1 and 2: p and U within the bound of tests/network_bound.py on the scale interval, U and p
      within OPS_TOL of the operator sequence (simulate.simulate) with the same zero bits, within MODE_TOL of
      oracle.simulate with the network in float64, and the density bit for bit against both.
  (2) Which path ran (torch.profiler, in a child interpreter as tests/step_cases.py explains): the fused input kernel
      of the block (4-voxel or per-voxel: an nx % 4 != 0 grid and unaligned views take the latter), the divergence
      statistics only for 'div', k_cnn_skip only with the skip, never the per-operator k_cnn_mask_stats,
      k_cnn_inputs_padded or k_cnn_scale; the launch tally equals the kernels the profiler saw.  A fp32-mode model
      and a state with pressure BCs take the operator sequence.
  (3) Batches: nb = 3 entries with their own flags, velocity and BCs, each equal to its scene stepped alone; the
      largest batch the launch grid holds runs and one entry more is refused by name before anything is launched.
  (4) A step graph replays direct steps bit for bit with in-place changes between replays; two identical runs give
      identical bits; the host-buffer step (tfl_host_sim_step) equals the device step."""
import ctypes as C

import numpy as np
import pytest
import torch

import oracle
from cases import bits_equal, describe_diff
from fluidnet_b200 import synth
from fluidnet_b200.model import ProjectionModel
from network_bound import check, projection_reference, tc_covered
from scenes import plume_batch
from step_cases import (MODE_TOL, OPS_TOL, close_per_entry, plume_bcs, quad_dims, run_in_child, same_zero_bits,
                        step_path)

pytestmark = pytest.mark.gpu

MCONF = oracle.default_mconf(dt=0.1, maccormackStrength=0.6, buoyancyScale=0.5, vorticityConfinementAmp=3.0,
                             simMethod="convnet")

# The input blocks of tests/test_gpu_cnn_network_f64.py.
INPUTS = {
    "all-channels": {"inputChannels": {"UDiv": True}},
    "udiv-only": {"inputChannels": {"pDiv": False, "UDiv": True, "div": False}},
    "norm": {"normalizeInputFunc": "norm"},
    "chan-pdiv": {"normalizeInputChan": "pDiv"},
    "chan-div": {"normalizeInputChan": "div"},
    "skip": {"addPressureSkip": True},
    "skip-udiv-norm": {"addPressureSkip": True, "inputChannels": {"UDiv": True}, "normalizeInputFunc": "norm"},
    "no-normalize": {"normalizeInput": False},
}
MODES = ("tf32x3", "tf32")
QUAD, SCALAR = (10, 12, 32), (9, 10, 30)       # the 4-voxel and the per-voxel kernels (nx % 4 != 0)


def fused_path(mnp, mode, pbc=False):
    """fused_step_applies (tfl_api.cu) for these 3-D convnet steps: a model the tensor cores cover, a tensor-core
    mode and no pressure BC, whatever the input block."""
    return tc_covered(mnp) and mode != "fp32" and not pbc


def model(case, mode):
    mnp = synth.make_model(True, inputs=INPUTS[case])
    gm = ProjectionModel.from_model(mnp)
    assert gm.get_mode() == "tf32x3"
    gm.set_mode(mode)
    assert fused_path(mnp, mode)
    return mnp, gm


def problem(shape, nb, seed=21):
    """A plume scene of nb entries (createPlumeBCs per entry) with a small signed pDiv."""
    batch = plume_batch(shape, nb=nb, seed=seed)
    plume_bcs(batch, nb)
    batch["pDiv"] = ((np.random.RandomState(seed).rand(*batch["flags"].shape) - 0.5) * 0.2).astype(np.float32)
    return {k: np.ascontiguousarray(v, np.float32) for k, v in batch.items()}


def gpu(batch, unaligned=False):
    out = {}
    for k, v in batch.items():
        t = torch.from_numpy(np.ascontiguousarray(v).copy()).cuda()
        if unaligned:                     # 4-byte aligned views: the per-voxel kernels run
            flat = torch.empty(t.numel() + 1, device="cuda", dtype=t.dtype)
            view = flat[1:].view(t.shape)
            view.copy_(t)
            assert view.data_ptr() % 16 == 4
            t = view
        out[k] = t
    return out


def host(batch):
    return {k: v.cpu().numpy() for k, v in batch.items()}


def step(st, gm, mconf=MCONF):
    from fluidnet_b200 import simulate
    simulate.simulate_fused(None, mconf, st, gm)


# ---------------------------------------------------------------------------------------------------------------
# (1) Per voxel against float64, the operator sequence and the oracle
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nb", [1, 2])
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", list(INPUTS))
def test_step_against_float64(orc, case, mode, nb):
    from fluidnet_b200 import simulate, tfluids
    mnp, gm = model(case, mode)
    batch = problem(QUAD, nb)
    fused, ops = gpu(batch), gpu(batch)
    bound = projection_reference(fused, MCONF, gm, mnp)
    ref = {k: v.copy() for k, v in batch.items()}
    oracle.simulate(orc, MCONF, ref, mnp, f64=True)
    ctx = tfluids.context()
    ctx.trace_faults()
    step(fused, gm)
    simulate.simulate(None, MCONF, ops, gm)
    got, opg = host(fused), host(ops)
    what = "fused step %s [%s] nb %d" % (case, mode, nb)
    rp = check(what + " p vs float64", got["pDiv"], bound["p"], bound["Ep"])
    rU = check(what + " U vs float64", got["UDiv"], bound["U"], bound["EU"])
    for name, want in (("ops", opg), ("oracle", ref)):
        assert bits_equal(got["density"], want["density"]), "%s density vs %s: %s" % (
            what, name, describe_diff(got["density"], want["density"]))
    for k in ("UDiv", "pDiv"):
        close_per_entry(got[k], opg[k], OPS_TOL, "%s %s vs ops" % (what, k))
        assert same_zero_bits(got[k], opg[k]), "%s %s: zeros differ from the operator sequence" % (what, k)
        close_per_entry(got[k], ref[k], MODE_TOL[mode], "%s %s vs oracle" % (what, k))
    assert ctx.trace_faults() == 0
    print("%s: max err/E p %.3g U %.3g" % (what, rp, rU))


# ---------------------------------------------------------------------------------------------------------------
# (2) Which path ran
# ---------------------------------------------------------------------------------------------------------------
def path_cases():
    """{id: (input block, mode, shape, unaligned, pressure BC)}."""
    out = {}
    for case in INPUTS:
        out["%s-quad" % case] = (case, "tf32x3", QUAD, False, False)
        out["%s-voxel" % case] = (case, "tf32x3", SCALAR, False, False)
    out["chan-pdiv-unaligned"] = ("chan-pdiv", "tf32", QUAD, True, False)
    out["skip-udiv-norm-unaligned"] = ("skip-udiv-norm", "tf32", QUAD, True, False)
    out["all-channels-fp32"] = ("all-channels", "fp32", QUAD, False, False)
    out["chan-div-pbc"] = ("chan-div", "tf32x3", QUAD, False, True)
    return out


def path_kernels():
    """{id: (launch tally, {kernel: count})} of one step per path case, under torch.profiler."""
    from fluidnet_b200 import tfluids
    from step_cases import tally_and_kernels
    out = {}
    for cid, (case, mode, shape, unaligned, pbc) in path_cases().items():
        gm = ProjectionModel.from_model(synth.make_model(True, inputs=INPUTS[case]))
        gm.set_mode(mode)
        batch = problem(shape, 1)
        if pbc:
            inv = np.ones_like(batch["flags"])
            inv[:, :, 2:5, 3:7, 4:9] = 0.0
            batch["pBCInvMask"] = inv
            batch["pBC"] = np.where(inv == 0, np.float32(0.05), np.float32(0.0)).astype(np.float32)
        st = gpu(batch, unaligned)
        tally, kernels = tally_and_kernels(tfluids.context(), lambda: step(st, gm), attempts=6)
        out[cid] = (tally, dict(kernels))
    return out


def test_fused_kernels_ran():
    seen = run_in_child("test_gpu_fused_inputs", "t.path_kernels()")
    cases = path_cases()
    assert set(seen) == set(cases)
    for cid, (case, mode, shape, unaligned, pbc) in cases.items():
        tally, kernels = seen[cid]
        names = sorted(kernels)
        has = lambda s: any(s in k for k in names)
        print("fused inputs %s: %d launches, %s" % (cid, tally, names))
        assert tally == sum(kernels.values()), (cid, tally, kernels)
        if not fused_path(synth.make_model(True, inputs=INPUTS[case]), mode, pbc):
            assert step_path(kernels) == "ops" and has("k_cnn_mask_stats") and not has("k_cnn_inputs_fused"), (cid, names)
            continue
        quad = quad_dims(1, *shape) is not None and not unaligned
        assert step_path(kernels) == ("quad" if quad else "scalar"), (cid, names)
        assert has("k_cnn_inputs_fused4" if quad else "k_cnn_inputs_fused<"), (cid, names)
        assert has("k_cnn_div_stats_fused") == (INPUTS[case].get("normalizeInputChan") == "div"), (cid, names)
        assert has("k_cnn_skip") == bool(INPUTS[case].get("addPressureSkip")), (cid, names)
        for op in ("k_cnn_mask_stats", "k_cnn_inputs_padded", "k_cnn_scale", "k_cnn_div_stats<", "k_cnn_finish<"):
            assert not has(op), (cid, op, names)


# ---------------------------------------------------------------------------------------------------------------
# (3) Batches
# ---------------------------------------------------------------------------------------------------------------
def scene3(orc, shape=(9, 12, 32)):
    """Three entries with their own flags (one open on its x and z faces), velocity (one at rest), pDiv, density and
    plume BCs; nb nz is odd, so quad blocks straddle two entries."""
    nz, ny, nx = shape
    flags = np.concatenate([synth.make_flags(nx, ny, nz, True, nb=1, geometry=True, seed=7 + b) for b in range(3)])
    flags[1, :, :, 1:-1, 0] = synth.FLUID
    flags[1, :, :, 1:-1, -1] = synth.FLUID
    flags[1, :, 0, 1:-1, :] = synth.FLUID
    flags[1, :, -1, 1:-1, :] = synth.FLUID
    U = np.concatenate([synth.make_smooth_velocity(flags[b:b + 1], True, amp=a, seed=31 + b) * np.float32(a > 0.01)
                        for b, a in enumerate((3.0, 8.0, 0.001))])
    orc.setWallBcsForward(U, flags)
    batch = {"pDiv": (synth.make_density(flags, seed=38) - np.float32(0.5)) * np.float32(0.1), "UDiv": U,
             "flags": flags, "density": synth.make_density(flags, seed=39)}
    plume_bcs(batch, 3)
    return {k: np.ascontiguousarray(v, np.float32) for k, v in batch.items()}


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", ["chan-pdiv", "chan-div", "skip-udiv-norm", "no-normalize", "udiv-only"])
def test_batch_entries_equal_their_scene_alone(orc, case, mode):
    _, gm = model(case, mode)
    batch = scene3(orc)
    st = gpu(batch)
    for s in range(2):
        before = host(st)
        step(st, gm)
        got = host(st)
        for b in range(3):
            one = gpu({k: v[b:b + 1] for k, v in before.items()})
            step(one, gm)
            one = host(one)
            what = "%s [%s] step %d entry %d" % (case, mode, s, b)
            assert bits_equal(got["density"][b:b + 1], one["density"]), what + " density"
            for k in ("UDiv", "pDiv"):
                close_per_entry(got[k][b:b + 1], one[k], OPS_TOL, "%s %s vs alone" % (what, k))
                assert same_zero_bits(got[k][b:b + 1], one[k]), "%s %s zeros" % (what, k)


def test_largest_batch_runs_and_one_more_is_refused(orc):
    from fluidnet_b200 import tfluids
    from fluidnet_b200._lib import TflError
    shape = (5, 8, 8)
    nb = 2 * 65535 // shape[0]                    # nb nz <= 2 x 65535 (check_launch_grid)
    _, gm = model("skip-udiv-norm", "tf32x3")
    proto = problem(shape, 1, seed=5)
    alone = gpu(proto)
    step(alone, gm)
    alone = host(alone)
    ctx = tfluids.context()

    def repeated(n):
        return {k: torch.from_numpy(v).cuda().repeat(n, 1, 1, 1, 1).contiguous() for k, v in proto.items()}

    st = repeated(nb)
    step(st, gm)
    for k in ("density", "UDiv", "pDiv"):
        rows = st[k].cpu().numpy().reshape(nb, -1).astype(np.float64)
        want = alone[k].reshape(1, -1).astype(np.float64)
        err = np.abs(rows - want).max()
        assert err <= OPS_TOL * max(np.abs(want).max(), 1e-6), (k, err)
    del st
    big = repeated(nb + 1)
    before = {k: v.clone() for k, v in big.items()}
    n0 = ctx.launch_count()
    with pytest.raises(TflError, match="at most %d" % (2 * 65535)):
        step(big, gm)
    torch.cuda.synchronize()
    assert ctx.launch_count() == n0
    assert all(torch.equal(big[k].view(torch.int32), before[k].view(torch.int32)) for k in big)


# ---------------------------------------------------------------------------------------------------------------
# (4) Graphs, repeatability, the host-buffer step
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["chan-div", "skip-udiv-norm", "chan-pdiv"])
def test_graph_replays_equal_direct_steps(orc, case):
    from fluidnet_b200 import simulate
    _, gm = model(case, "tf32x3")
    batch = scene3(orc)
    stream = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(stream):
        direct, replayed = gpu(batch), gpu(batch)
        step(direct, gm)
        step(replayed, gm)
        graph = simulate.StepGraph(MCONF, replayed, gm)
        try:
            for s in range(4):
                if s >= 2:                 # in-place changes between replays reach the captured tensors
                    for st in (direct, replayed):
                        st["density"][1].mul_(0.5)
                        st["UDiv"][0].mul_(-1.0 if s == 2 else 1.5)
                        st["pDiv"][-1].mul_(-2.0)
                step(direct, gm)
                graph.launch()
                stream.synchronize()
                for k in ("pDiv", "UDiv", "density"):
                    a, b = direct[k].cpu().numpy(), replayed[k].cpu().numpy()
                    assert bits_equal(a, b), "%s replay %d %s: %s" % (case, s, k, describe_diff(b, a))
        finally:
            graph.close()


@pytest.mark.parametrize("case", list(INPUTS))
def test_two_runs_give_the_same_bits(case):
    _, gm = model(case, "tf32x3")
    batch = problem((16, 16, 64), 2, seed=3)
    runs = []
    for _ in range(2):
        st = gpu(batch)
        for _ in range(3):
            step(st, gm)
        runs.append(host(st))
    for k in ("pDiv", "UDiv", "density"):
        assert bits_equal(runs[0][k], runs[1][k]), "%s %s: %s" % (case, k, describe_diff(runs[1][k], runs[0][k]))


@pytest.mark.parametrize("case", ["chan-pdiv", "chan-div", "skip-udiv-norm"])
def test_host_buffer_step_equals_the_device_step(case):
    from fluidnet_b200 import simulate, tfluids
    _, gm = model(case, "tf32x3")
    nz, ny, nx = QUAD
    batch = problem(QUAD, 1)
    dev = gpu(batch)
    ctx = tfluids.context()
    lib = ctx.lib
    hs = C.c_void_p()
    keep = [np.ascontiguousarray(batch[k]) for k in ("flags", "UBC", "UBCInvMask", "densityBC", "densityBCInvMask")]
    ctx.check(lib.tfl_host_sim_create(ctx.h, 1, nz, ny, nx, 1, *[a.ctypes.data for a in keep], C.byref(hs)))
    hp, hU, hd = (torch.from_numpy(batch[k].copy()).pin_memory() for k in ("pDiv", "UDiv", "density"))
    mc = simulate.make_mconf(MCONF)
    try:
        for s in range(2):
            step(dev, gm)
            ctx.check(lib.tfl_host_sim_step(ctx.h, hs, hp.data_ptr(), hU.data_ptr(), hd.data_ptr(), C.byref(mc), gm.h))
            for k, h in (("density", hd), ("UDiv", hU), ("pDiv", hp)):
                a, b = dev[k].cpu().numpy(), h.numpy()
                assert bits_equal(a, b), "%s step %d %s: %s" % (case, s, k, describe_diff(b, a))
    finally:
        lib.tfl_host_sim_destroy(ctx.h, hs)
