"""Whole-step parity: tfluids.simulate (torch/lib/simulate.lua:175-327) on the GPU, both
operator-by-operator (fluidnet_b200.simulate.simulate) and through the single C-ABI call
(tfl_simulate_step), against the oracle's restatement of the same loop.

Tolerances
  * jacobi path (no conv): bit-exact -- every kernel is a per-cell restatement built
    without FMA contraction.
  * convnet path: the conv stack accumulates in fp32 FMA on the GPU and in fp64 in the
    oracle (the reference used cuDNN, algorithm unspecified): |err| <= 2e-5 * max|field|
    after one step, the reference's own cross-backend tolerance class (1e-5 abs on O(1)
    data, test_tfluids.lua:34).  The input scale (sample std) is a reduction: 1e-5 rel."""
import numpy as np
import pytest
import torch

import oracle
from cases import bits_equal, describe_diff
from fluidnet_b200 import synth

pytestmark = pytest.mark.gpu


def make_batch(n, is3d, plume=True, geometry=True, amp=3.0, shape=None, nb=1, seed=1234):
    """An n^2 / n^3 grid, or shape = (nz, ny, nx); with nb > 1 every entry has its own velocity field."""
    nz, ny, nx = shape if shape is not None else ((n if is3d else 1), n, n)
    flags = synth.make_flags(nx, ny, nz, is3d, nb=nb, geometry=geometry)
    U = synth.make_smooth_velocity(flags, is3d, amp=amp, seed=seed)
    oracle.Oracle().setWallBcsForward(U, flags)
    batch = {"pDiv": np.zeros_like(flags), "UDiv": U, "flags": flags, "density": synth.make_density(flags)}
    if plume:
        oracle.create_plume_bcs(batch, [1.0], nx / 128.0 * 4, 0.15)
    return batch


def to_gpu(batch):
    return {k: torch.from_numpy(v.copy()).cuda() for k, v in batch.items() if v is not None}


def close(got, want, tol, what):
    err = np.abs(got.astype(np.float64) - want.astype(np.float64)).max()
    scale = max(np.abs(want).max(), 1e-6)
    assert err <= tol * scale, "%s: max err %g vs scale %g" % (what, err, scale)


@pytest.mark.parametrize("is3d,n", [(False, 64), (True, 20)], ids=["2d64", "3d20"])
@pytest.mark.parametrize("fused", [False, True], ids=["ops", "fused"])
def test_step_jacobi_bit_exact(orc, is3d, n, fused):
    """BASELINE config 1: 2-D 64x64 smoke, Jacobi projection, 1 step (and a small 3-D one)."""
    from fluidnet_b200 import simulate
    batch = make_batch(n, is3d)
    mconf = oracle.default_mconf(dt=0.1, maccormackStrength=0.6, buoyancyScale=1.0,
                                 vorticityConfinementAmp=(0.0 if not is3d else 3.0),
                                 simMethod="jacobi", maxIter=100, is3D=is3d)
    gb = to_gpu(batch)
    for step in range(2):
        (simulate.simulate_fused if fused else simulate.simulate)(None, mconf, gb, None)
        oracle.simulate(orc, mconf, batch, None)
        for k in ("density", "UDiv", "pDiv"):
            got = gb[k].cpu().numpy()
            assert bits_equal(got, batch[k]), "step %d %s: %s" % (step, k, describe_diff(got, batch[k]))


# conv arithmetic -> tolerance relative to max|field| (see module docstring; tf32 = single-pass
# TF32 tensor cores, 10-bit mantissa inputs, is the "fast" mode and NOT the default)
MODE_TOL = {"fp32": 2e-5, "tf32x3": 2e-5, "tf32": 3e-3}


FORWARD_CASES = {          # id: (is3d, (nz, ny, nx), nb, mode, zero_u_entry)
    "3d24-fp32": (True, (24, 24, 24), 1, "fp32", None),
    "3d24-tf32x3": (True, (24, 24, 24), 1, "tf32x3", None),
    "3d24-tf32": (True, (24, 24, 24), 1, "tf32", None),
    "3d37-tf32x3": (True, (37, 37, 37), 1, "tf32x3", None),
    "3d37-tf32": (True, (37, 37, 37), 1, "tf32", None),
    "2d48-fp32": (False, (1, 48, 48), 1, "fp32", None),
    # non-cubic, nb = 2: odd nz (per-thread atomics in k_cnn_mask_stats) and even nz (block sums)
    "3d13x18x23-nb2-fp32": (True, (13, 18, 23), 2, "fp32", None),
    "3d13x18x23-nb2-tf32x3": (True, (13, 18, 23), 2, "tf32x3", None),
    "3d13x18x23-nb2-tf32": (True, (13, 18, 23), 2, "tf32", None),
    "3d10x21x34-nb2-fp32": (True, (10, 21, 34), 2, "fp32", None),
    "3d10x21x34-nb2-tf32x3": (True, (10, 21, 34), 2, "tf32x3", None),
    "3d10x21x34-nb2-tf32": (True, (10, 21, 34), 2, "tf32", None),
    # entry 0 has UDiv = 0, so its input scale clamps to the threshold; entry 1 does not
    "3d12x16x20-nb2-zeroU-tf32x3": (True, (12, 16, 20), 2, "tf32x3", 0),
    "2d40x56-nb2-fp32": (False, (1, 40, 56), 2, "fp32", None),
}


@pytest.mark.parametrize("case", list(FORWARD_CASES))
def test_cnn_projection_forward(orc, case):
    """BASELINE config 2 (shape-reduced for the CPU oracle): model:forward only, for every
    arithmetic mode of the conv stack (37^3 exercises partial tensor-core tiles), on non-cubic grids and
    batches of two.  Each batch entry is checked on its own: its scale, and p / U relative to its own max."""
    from gpu_backend import make_gpu_model
    is3d, shape, nb, mode, zero_u = FORWARD_CASES[case]
    batch = make_batch(0, is3d, plume=False, shape=shape, nb=nb)
    if zero_u is not None:
        batch["UDiv"][zero_u] = 0.0
    mnp = synth.make_model(is3d)
    p0 = (synth.make_density(batch["flags"], seed=77) - np.float32(0.5)) * np.float32(0.1)
    wp, wU, wscale = oracle.model_forward(orc, mnp, p0, batch["UDiv"], batch["flags"])
    gm = make_gpu_model(mnp)
    assert gm.get_mode() == ("tf32x3" if is3d else "fp32")      # defaults
    gm.set_mode(mode)
    gp, gU = gm.forward((torch.from_numpy(p0).cuda(), torch.from_numpy(batch["UDiv"]).cuda(),
                         torch.from_numpy(batch["flags"]).cuda()), return_scale=True)
    gp, gU = gp.cpu().numpy(), gU.cpu().numpy()
    if zero_u is not None:
        assert wscale[zero_u] == np.float32(1e-5) and wscale[1 - zero_u] > np.float32(1e-5)
    for b in range(nb):
        assert abs(gm.last_scale[b] - wscale[b]) <= 1e-5 * wscale[b], (b, gm.last_scale, wscale)
        close(gp[b], wp[b], MODE_TOL[mode], "p[%d]" % b)
        close(gU[b], wU[b], MODE_TOL[mode], "U[%d]" % b)
    # occupancy / wall logic is exact: every face the oracle zeroes is exactly zero here.
    assert np.array_equal(gU == 0, wU == 0)


def test_cnn_model_state_across_shapes_and_modes():
    """One model through grid changes (each reallocates its padded activation buffers), mode changes and new
    inputs on the same grid: every result equals that of a fresh model for the same shape and mode, so the zero
    borders of the activation buffers survive between calls."""
    from gpu_backend import make_gpu_model
    mnp = synth.make_model(True)
    A, B = ((12, 16, 20), 1), ((9, 13, 31), 2)
    gm = make_gpu_model(mnp)
    for (shape, nb), mode, seed in ((A, "tf32x3", 0), (B, "tf32", 0), (A, "fp32", 0), (A, "tf32x3", 1),
                                    (A, "tf32x3", 2), (B, "tf32x3", 1)):
        batch = make_batch(0, True, plume=False, shape=shape, nb=nb, seed=1234 + seed)
        p0 = (synth.make_density(batch["flags"], seed=77 + seed) - np.float32(0.5)) * np.float32(0.1)
        inputs = (torch.from_numpy(p0).cuda(), torch.from_numpy(batch["UDiv"]).cuda(),
                  torch.from_numpy(batch["flags"]).cuda())
        gm.set_mode(mode)
        fresh = make_gpu_model(mnp)
        fresh.set_mode(mode)
        what = "%s nb%d %s seed %d" % (shape, nb, mode, seed)
        for got, want, k in zip(gm.forward(inputs), fresh.forward(inputs), ("p", "U")):
            close(got.cpu().numpy(), want.cpu().numpy(), 1e-6, "%s %s" % (what, k))


@pytest.mark.parametrize("fused", [False, True], ids=["ops", "fused"])
def test_step_convnet(orc, fused):
    """BASELINE config 3 shape-reduced: CNN projection + vorticity confinement + MacCormack."""
    from fluidnet_b200 import simulate
    from gpu_backend import make_gpu_model
    n = 24
    batch = make_batch(n, True)
    mnp = synth.make_model(True)
    gm = make_gpu_model(mnp)
    mconf = oracle.default_mconf(dt=0.1, maccormackStrength=0.6, buoyancyScale=2.0 * n / 128,
                                 vorticityConfinementAmp=3.0, simMethod="convnet")
    gb = to_gpu(batch)
    for step in range(2):
        (simulate.simulate_fused if fused else simulate.simulate)(None, mconf, gb, gm)
        oracle.simulate(orc, mconf, batch, mnp)
        tol = 2e-5 if step == 0 else 2e-4          # second step: advection of slightly different fields
        for k in ("density", "UDiv", "pDiv"):
            close(gb[k].cpu().numpy(), batch[k], tol, "step %d %s" % (step, k))


def test_fused_equals_operator_sequence():
    """tfl_simulate_step must equal calling the operators one by one (bitwise)."""
    from fluidnet_b200 import simulate
    from gpu_backend import make_gpu_model
    n = 32
    batch = make_batch(n, True)
    gm = make_gpu_model(synth.make_model(True))
    mconf = oracle.default_mconf(dt=0.1, maccormackStrength=0.6, buoyancyScale=0.5,
                                 vorticityConfinementAmp=3.0, simMethod="convnet")
    a, b = to_gpu(batch), to_gpu(batch)
    for _ in range(3):
        simulate.simulate(None, mconf, a, gm)
        simulate.simulate_fused(None, mconf, b, gm)
    for k in ("density", "UDiv", "pDiv"):
        # the only non-deterministic piece is the double-precision atomic sum behind the
        # input scale; allow 1 ulp-class differences there.
        close(a[k].cpu().numpy(), b[k].cpu().numpy(), 1e-6, k)


@pytest.mark.parametrize("method", ["convnet", "jacobi"])
def test_host_buffer_step_equals_device_step(method):
    """tfl_host_sim_step (pinned host buffers in and out, the copies overlapped with the fused step)
    returns what tfl_simulate_step leaves on the device, over several steps."""
    import ctypes as C
    import torch
    from fluidnet_b200 import simulate, tfluids
    from gpu_backend import make_gpu_model
    n = 32
    batch = make_batch(n, True)
    gm = make_gpu_model(synth.make_model(True))
    mconf = oracle.default_mconf(dt=0.1, maccormackStrength=0.6, buoyancyScale=0.5,
                                 vorticityConfinementAmp=3.0, simMethod=method, maxIter=20)
    dev_batch = to_gpu(batch)
    ctx = tfluids.context()
    lib = ctx.lib
    hs = C.c_void_p()
    keep = [np.ascontiguousarray(batch[k]) for k in ("flags", "UBC", "UBCInvMask", "densityBC", "densityBCInvMask")]
    ctx.check(lib.tfl_host_sim_create(ctx.h, 1, n, n, n, 1, *[a.ctypes.data for a in keep], C.byref(hs)))
    hp = torch.from_numpy(batch["pDiv"].copy()).pin_memory()
    hU = torch.from_numpy(batch["UDiv"].copy()).pin_memory()
    hd = torch.from_numpy(batch["density"].copy()).pin_memory()
    mc = simulate.make_mconf(mconf)
    try:
        for step in range(3):
            simulate.simulate_fused(None, mconf, dev_batch, gm)
            ctx.check(lib.tfl_host_sim_step(ctx.h, hs, hp.data_ptr(), hU.data_ptr(), hd.data_ptr(), C.byref(mc), gm.h))
            for k, h in (("density", hd), ("UDiv", hU), ("pDiv", hp)):
                close(h.numpy(), dev_batch[k].cpu().numpy(), 1e-6, "step %d %s" % (step, k))
    finally:
        lib.tfl_host_sim_destroy(ctx.h, hs)


def test_trained_reference_model_2d(orc):
    """The 2-D model the reference ships (data/models/myModel2D, read by fluidnet_b200/torch7.py; weights
    committed as tests/golden/myModel2D_layers.npz): model:forward and three simulate steps with its
    own mconf (maccormack advection, no buoyancy), against the oracle.  A trained projection must also do
    its job: it leaves less divergence than it was given."""
    import os
    from fluidnet_b200 import simulate
    from gpu_backend import make_gpu_model
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "myModel2D_layers.npz"))
    mnp = {"is3D": bool(z["is3D"]), "layers": [(z["w%d" % i], z["b%d" % i]) for i in range(int(z["n_layers"]))]}
    assert mnp["is3D"] is False
    n = 64
    batch = make_batch(n, False, plume=False, amp=1.0)
    gm = make_gpu_model(mnp, threshold=float(z["normalizeInputThreshold"]))
    p0 = np.zeros_like(batch["flags"])
    wp, wU, wscale = oracle.model_forward(orc, mnp, p0, batch["UDiv"], batch["flags"])
    gp, gU = gm.forward((torch.from_numpy(p0).cuda(), torch.from_numpy(batch["UDiv"]).cuda(),
                         torch.from_numpy(batch["flags"]).cuda()), return_scale=True)
    close(gp.cpu().numpy(), wp, 2e-5, "p")
    close(gU.cpu().numpy(), wU, 2e-5, "U")
    div_in = np.linalg.norm(orc.velocityDivergenceForward(batch["UDiv"], batch["flags"]))
    div_out = np.linalg.norm(orc.velocityDivergenceForward(gU.cpu().numpy(), batch["flags"]))
    assert div_out < 0.8 * div_in, (div_in, div_out)       # (this small model removes ~40 % per application)
    mconf = oracle.default_mconf(dt=0.1, advectionMethod="maccormack", maccormackStrength=0.75, is3D=False,
                                 simMethod="convnet")
    gb = to_gpu(batch)
    for step in range(3):
        simulate.simulate(None, mconf, gb, gm)
        oracle.simulate(orc, mconf, batch, mnp)
        for k in ("density", "UDiv", "pDiv"):
            close(gb[k].cpu().numpy(), batch[k], 2e-5 * (step + 1) * 5, "step %d %s" % (step, k))


@pytest.mark.parametrize("is3d,n,model_type,pool_type", [(False, 48, "tog", "avg"), (True, 24, "tog", "avg"),
                                                          (True, 16, "tog", "max"), (False, 40, "yang", "avg"),
                                                          (True, 20, "yang", "avg")],
                         ids=["2d-tog", "3d-tog", "3d-tog-max", "2d-yang", "3d-yang"])
def test_cnn_model_graphs(orc, is3d, n, model_type, pool_type):
    """The other single-bank graphs of lib/model.lua:164-226: 'tog' (pooling, ConvolutionUpsample pixel
    shuffles, 5x5 / 1x1 / 256-channel convolutions) and 'yang' (sigmoid), model:forward against the oracle
    (whose graph semantics are pinned on torch.nn.functional, tests/test_oracle_model_graph.py)."""
    from gpu_backend import make_gpu_model
    batch = make_batch(n, is3d, plume=False)
    mnp = synth.make_model(is3d, model_type=model_type)
    if model_type == "tog":
        mnp["poolType"] = pool_type
    p0 = (synth.make_density(batch["flags"], seed=77) - np.float32(0.5)) * np.float32(0.1)
    wp, wU, wscale = oracle.model_forward(orc, mnp, p0, batch["UDiv"], batch["flags"])
    gm = make_gpu_model(mnp)
    assert gm.get_mode() == "fp32"
    gp, gU = gm.forward((torch.from_numpy(p0).cuda(), torch.from_numpy(batch["UDiv"]).cuda(),
                         torch.from_numpy(batch["flags"]).cuda()), return_scale=True)
    assert abs(gm.last_scale[0] - wscale[0]) <= 1e-5 * wscale[0]
    close(gp.cpu().numpy(), wp, 2e-5, "p")
    close(gU.cpu().numpy(), wU, 2e-5, "U")


def test_cnn_graph_argument_errors():
    from fluidnet_b200 import model as fmodel
    from fluidnet_b200._lib import TflError
    m = synth.make_model(True, model_type="tog")
    with pytest.raises(TflError, match="same layer"):
        fmodel.ProjectionModel(m["layers"], True, pool=[2, 2, 1, 1, 1, 2, 1], up=m["up"])
    with pytest.raises(TflError, match="input resolution"):
        fmodel.ProjectionModel(m["layers"], True, pool=[2, 1, 1, 1, 1, 1, 1], up=m["up"])
    gm = fmodel.ProjectionModel(m["layers"], True, pool=m["pool"], up=m["up"])
    f = torch.ones(1, 1, 6, 8, 8, device="cuda")               # 6 is not divisible by the two 2x poolings
    with pytest.raises(TflError, match="divisible"):
        gm.forward((torch.zeros_like(f), torch.zeros(1, 3, 6, 8, 8, device="cuda"), f))


def test_full_size_properties():
    """BASELINE-size (128^3) checks that do not need the CPU oracle: the Jacobi-projected
    velocity is (nearly) divergence free, the obstacle faces stay exactly zero, advection of
    a constant field is the identity in the fluid interior, and nothing traces out of bounds."""
    from fluidnet_b200 import tfluids
    n = 128
    flags_np = synth.make_flags(n, n, n, True, nb=1, geometry=True)
    flags = torch.from_numpy(flags_np).cuda()
    U = torch.from_numpy(synth.make_smooth_velocity(flags_np, True, amp=4.0)).cuda()
    tfluids.setWallBcsForward(U, flags)
    ones = torch.where(flags == 1, 1.0, 0.0).contiguous()
    adv = torch.empty_like(ones)
    tfluids.advectScalar(0.1, ones, U, flags, "maccormackOurs", adv, False, 0.6)
    interior = torch.zeros_like(flags, dtype=torch.bool)
    interior[..., 1:-1, 1:-1, 1:-1] = True
    fluid_in = (flags == 1) & interior
    assert torch.all(adv[fluid_in] == 1.0)           # interpolating only fluid cells of a constant
    div = torch.empty_like(flags)
    tfluids.velocityDivergenceForward(U, flags, div)
    d0 = div.abs().max().item()
    p = torch.zeros_like(flags)
    tfluids.solveLinearSystemJacobi(p, flags, div, True, 0, 2000)
    tfluids.velocityUpdateForward(U, flags, p)
    tfluids.setWallBcsForward(U, flags)
    tfluids.velocityDivergenceForward(U, flags, div)
    assert div.abs().max().item() < 0.2 * d0
    # idempotence of the wall BCs
    U2 = U.clone()
    tfluids.setWallBcsForward(U2, flags)
    assert torch.equal(U, U2)
    assert tfluids.context().trace_faults() == 0


def test_fused_step_with_non_idempotent_density_bc():
    """setConstVals runs three times per step (lib/simulate.lua:202, :252, :321).  With an additive density
    BC (invMask = 1 where bc != 0) the three applications do not collapse into one: the fused step must still
    equal the operator sequence."""
    from fluidnet_b200 import simulate
    from gpu_backend import make_gpu_model
    n = 32
    batch = make_batch(n, True)
    rs = np.random.RandomState(5)
    batch["densityBC"] = (rs.rand(*batch["density"].shape) < 0.1).astype(np.float32) * np.float32(0.25)
    batch["densityBCInvMask"] = np.where(rs.rand(*batch["density"].shape) < 0.5, 1.0, 0.5).astype(np.float32)
    gm = make_gpu_model(synth.make_model(True))
    mconf = oracle.default_mconf(dt=0.1, maccormackStrength=0.6, buoyancyScale=0.5,
                                 vorticityConfinementAmp=3.0, simMethod="convnet")
    a, b = to_gpu(batch), to_gpu(batch)
    for _ in range(2):
        simulate.simulate(None, mconf, a, gm)
        simulate.simulate_fused(None, mconf, b, gm)
    assert bits_equal(a["density"].cpu().numpy(), b["density"].cpu().numpy())
    for k in ("UDiv", "pDiv"):
        close(a[k].cpu().numpy(), b[k].cpu().numpy(), 1e-6, k)


def test_fused_step_on_unaligned_views():
    """Caller-owned grids that are contiguous but only 4-byte aligned (a view with an odd storage offset):
    the 16-byte kernels must step aside, results equal the aligned run bit for bit."""
    from fluidnet_b200 import simulate
    from gpu_backend import make_gpu_model
    n = 32
    batch = make_batch(n, True)
    gm = make_gpu_model(synth.make_model(True))
    mconf = oracle.default_mconf(dt=0.1, maccormackStrength=0.6, buoyancyScale=0.5,
                                 vorticityConfinementAmp=3.0, simMethod="convnet")
    a = to_gpu(batch)
    b = {}
    for k, v in to_gpu(batch).items():
        flat = torch.empty(v.numel() + 1, device="cuda", dtype=v.dtype)
        view = flat[1:].view(v.shape)
        view.copy_(v)
        assert view.data_ptr() % 16 == 4 and view.is_contiguous()
        b[k] = view
    simulate.simulate_fused(None, mconf, a, gm)
    simulate.simulate_fused(None, mconf, b, gm)
    torch.cuda.synchronize()
    assert bits_equal(a["density"].cpu().numpy(), b["density"].cpu().numpy())
    for k in ("UDiv", "pDiv"):
        close(a[k].cpu().numpy(), b[k].cpu().numpy(), 1e-6, k)


def test_operators_on_a_non_current_device(orc):
    """Contexts select their own device: tensors on cuda:1 while the current device is cuda:0 (needs 2 GPUs)."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from fluidnet_b200 import tfluids
    c = make_batch(20, True, plume=False)
    want = orc.advectVel(0.1, c["UDiv"], c["flags"], "maccormackOurs", 0.6)
    torch.cuda.set_device(0)
    U = torch.from_numpy(c["UDiv"]).to("cuda:1")
    fl = torch.from_numpy(c["flags"]).to("cuda:1")
    out = torch.empty_like(U)
    tfluids.advectVel(0.1, U, fl, "maccormackOurs", out, 0.6)
    assert torch.cuda.current_device() == 0
    assert bits_equal(out.cpu().numpy(), want)
    div = torch.empty_like(fl)
    tfluids.velocityDivergenceForward(U, fl, div)
    assert bits_equal(div.cpu().numpy(), orc.velocityDivergenceForward(c["UDiv"], c["flags"]))


def test_step_as_cuda_graph_equals_direct_step(orc):
    """tfl_step_graph_*: the fused step captured once and replayed gives the bits of the direct call (same
    kernels), on the convnet and on the Jacobi path; capturing on the default stream is refused."""
    import torch
    from fluidnet_b200 import simulate, synth
    from fluidnet_b200._lib import TflError
    from gpu_backend import make_gpu_model
    n = 32
    flags = synth.make_flags(n, n, n, True, nb=1, geometry=True)
    U = synth.make_smooth_velocity(flags, True, amp=3.0)
    orc.setWallBcsForward(U, flags)
    batch = {"pDiv": np.zeros_like(flags), "UDiv": U, "flags": flags, "density": synth.make_density(flags)}
    oracle.create_plume_bcs(batch, [1.0], n / 128.0, 0.15)
    mnp = synth.make_model(True)
    for sim_method, model in (("convnet", make_gpu_model(mnp)), ("jacobi", None)):
        mconf = oracle.default_mconf(dt=0.1, maccormackStrength=0.6, buoyancyScale=2.0 * n / 128,
                                     vorticityConfinementAmp=3.0, simMethod=sim_method, maxIter=12)
        ga = {k: torch.from_numpy(v.copy()).cuda() for k, v in batch.items()}
        gb = {k: torch.from_numpy(v.copy()).cuda() for k, v in batch.items()}
        with pytest.raises(TflError):
            simulate.simulate_fused(None, mconf, gb, model)       # sizes the scratch buffers ...
            simulate.StepGraph(mconf, gb, model)                  # ... but the default stream cannot be captured
        gb = {k: torch.from_numpy(v.copy()).cuda() for k, v in batch.items()}
        stream = torch.cuda.Stream()
        torch.cuda.synchronize()
        with torch.cuda.stream(stream):
            simulate.simulate_fused(None, mconf, ga, model)
            simulate.simulate_fused(None, mconf, gb, model)
            graph = simulate.StepGraph(mconf, gb, model)          # capture executes nothing
            for _ in range(2):
                simulate.simulate_fused(None, mconf, ga, model)
                graph.launch()
            stream.synchronize()
            for k in ("density", "UDiv", "pDiv"):
                assert torch.equal(ga[k].view(torch.int32), gb[k].view(torch.int32)), (sim_method, k)
            graph.close()
