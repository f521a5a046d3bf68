"""Parity at the shapes BASELINE.json names, on the kernels bench.py times.

The per-operator tests use edges of 14-40 cells; the bench runs 64^3 / 128^3 grids, where other kernel
variants are selected by shape (4-voxels-per-thread point-wise stages, tensor-core conv rows,
64-wide advection blocks, the clear-space advection path over a large obstacle-free interior).  These
tests put exactly those launches against the CPU oracle (which finishes a 128^3 operator in < 2 s):

  C2  64^3  model:forward, every arithmetic mode of the conv stack          (2e-5 / 3e-3, stated per mode)
  C3  128^3 one fused step: maccormackOurs + buoyancy + vorticity + CNN     (advected fields bit-exact,
                                                                             projected fields 2e-5)
  C4  128^3 100 Jacobi sweeps                                                (p bit-exact)
  advectVel / advectScalar at 128^3 with geometry                            (bit-exact)
  32^3 / 64^3 fused convnet steps: the quad kernels against the oracle directly
"""
import numpy as np
import pytest
import torch

import oracle
from cases import bits_equal, describe_diff
from fluidnet_b200 import synth

pytestmark = pytest.mark.gpu


def close(got, want, tol, what):
    err = np.abs(got.astype(np.float64) - want.astype(np.float64)).max()
    scale = max(np.abs(want).max(), 1e-6)
    assert err <= tol * scale, "%s: max err %g vs scale %g" % (what, err, scale)


def make_batch(n, plume=True, amp=3.0, smooth=True):
    flags = synth.make_flags(n, n, n, True, nb=1, geometry=True)
    U = (synth.make_smooth_velocity if smooth else synth.make_velocity)(flags, True, amp=amp)
    oracle.Oracle().setWallBcsForward(U, flags)
    batch = {"pDiv": np.zeros_like(flags), "UDiv": U, "flags": flags, "density": synth.make_density(flags)}
    if plume:
        oracle.create_plume_bcs(batch, [1.0], n / 128.0, 0.15)
    return batch


def to_gpu(batch):
    return {k: torch.from_numpy(v.copy()).cuda() for k, v in batch.items() if v is not None}


@pytest.fixture(scope="module")
def gpu():
    from gpu_backend import GpuBackend
    return GpuBackend()


MODE_TOL = {"fp32": 2e-5, "tf32x3": 2e-5, "tf32": 3e-3}


@pytest.mark.parametrize("mode", ["fp32", "tf32x3", "tf32"])
def test_c2_model_forward_64(orc, mode):
    """BASELINE config 2: 3-D 64^3, CNN pressure projection forward."""
    from gpu_backend import make_gpu_model
    batch = make_batch(64, plume=False)
    mnp = synth.make_model(True)
    p0 = (synth.make_density(batch["flags"], seed=77) - np.float32(0.5)) * np.float32(0.1)
    wp, wU, wscale = oracle.model_forward(orc, mnp, p0, batch["UDiv"], batch["flags"])
    gm = make_gpu_model(mnp)
    gm.set_mode(mode)
    gp, gU = gm.forward((torch.from_numpy(p0).cuda(), torch.from_numpy(batch["UDiv"]).cuda(),
                         torch.from_numpy(batch["flags"]).cuda()), return_scale=True)
    assert abs(gm.last_scale[0] - wscale[0]) <= 1e-5 * wscale[0]
    close(gp.cpu().numpy(), wp, MODE_TOL[mode], "p")
    close(gU.cpu().numpy(), wU, MODE_TOL[mode], "U")
    assert np.array_equal(gU.cpu().numpy() == 0, wU == 0)


@pytest.mark.parametrize("n", [32, 64, 128])
def test_c3_fused_step_vs_oracle(orc, n):
    """BASELINE config 3 (n = 128) and the smaller cubes whose rows also select the 4-voxel kernels: the
    single-call fused step against oracle.simulate.  The density leaves the step after the advection and
    the boundary conditions only -> bit-exact; U and p pass through the conv stack -> 2e-5 (3xTF32)."""
    from fluidnet_b200 import simulate
    from gpu_backend import make_gpu_model
    batch = make_batch(n)
    mnp = synth.make_model(True)
    gm = make_gpu_model(mnp)
    assert gm.get_mode() == "tf32x3"
    mconf = oracle.default_mconf(dt=0.1, maccormackStrength=0.6, buoyancyScale=2.0 * n / 128,
                                 vorticityConfinementAmp=3.0, simMethod="convnet")
    gb = to_gpu(batch)
    simulate.simulate_fused(None, mconf, gb, gm)
    torch.cuda.synchronize()
    oracle.simulate(orc, mconf, batch, mnp)
    got = gb["density"].cpu().numpy()
    assert bits_equal(got, batch["density"]), "density: " + describe_diff(got, batch["density"])
    for k in ("UDiv", "pDiv"):
        close(gb[k].cpu().numpy(), batch[k], 2e-5, k)
    from fluidnet_b200 import tfluids
    assert tfluids.context().trace_faults() == 0


@pytest.mark.parametrize("amp,smooth", [(3.0, True), (2.0, False), (25.0, False)],
                         ids=["smooth3", "random2", "random25"])
def test_advection_128_bit_exact(orc, gpu, amp, smooth):
    """advectVel / advectScalar (maccormackOurs) on the 128^3 grid with the sphere + slab geometry: the
    large clear interior takes the clear-space path, cells near the solids and (amp 25: 2.5-cell traces)
    fast cells the general one."""
    b = make_batch(128, plume=False, amp=amp, smooth=smooth)
    U, fl, d = b["UDiv"], b["flags"], b["density"]
    want = orc.advectVel(0.1, U, fl, "maccormackOurs", 0.6)
    got = gpu.advectVel(0.1, U, fl, "maccormackOurs", 0.6)
    assert bits_equal(got, want), "advectVel " + describe_diff(got, want)
    for outside in (False, True):
        want = orc.advectScalar(0.1, d, U, fl, "maccormackOurs", outside, 0.6)
        got = gpu.advectScalar(0.1, d, U, fl, "maccormackOurs", outside, 0.6)
        assert bits_equal(got, want), "advectScalar " + describe_diff(got, want)
    want = orc.advectVel(0.1, U, fl, "eulerOurs", 0.6)
    got = gpu.advectVel(0.1, U, fl, "eulerOurs", 0.6)
    assert bits_equal(got, want), "advectVel eulerOurs " + describe_diff(got, want)
    assert gpu.trace_faults() == 0


def test_c4_jacobi_128_bit_exact(orc, gpu):
    """BASELINE config 4: divergence + 100 Jacobi sweeps + velocity update at 128^3."""
    b = make_batch(128, plume=False)
    U, fl = b["UDiv"], b["flags"]
    div_w = orc.velocityDivergenceForward(U, fl)
    div_g = gpu.velocityDivergenceForward(U, fl)
    assert bits_equal(div_g, div_w)
    a = np.full_like(div_w, 9.0)
    w = np.full_like(div_w, 9.0)
    ra = gpu.solveLinearSystemJacobi(a, fl, div_w, True, 0.0, 100)
    rb = orc.solveLinearSystemJacobi(w, fl, div_w, True, 0.0, 100)
    assert bits_equal(a, w), "jacobi p: " + describe_diff(a, w)
    assert abs(ra - rb) <= 1e-5 * max(abs(rb), 1e-12)
    Ua, Ub = U.copy(), U.copy()
    gpu.velocityUpdateForward(Ua, fl, a)
    orc.velocityUpdateForward(Ub, fl, w)
    assert bits_equal(Ua, Ub)


def test_jacobi_step_64_bit_exact(orc):
    """Whole step on the Jacobi path at 64^3 (every kernel a per-cell restatement): bit-exact."""
    from fluidnet_b200 import simulate
    batch = make_batch(64)
    mconf = oracle.default_mconf(dt=0.1, maccormackStrength=0.6, buoyancyScale=1.0,
                                 vorticityConfinementAmp=3.0, simMethod="jacobi", maxIter=30, is3D=True)
    gb = to_gpu(batch)
    for step in range(2):
        simulate.simulate_fused(None, mconf, gb, None)
        oracle.simulate(orc, mconf, batch, None)
        for k in ("density", "UDiv", "pDiv"):
            got = gb[k].cpu().numpy()
            assert bits_equal(got, batch[k]), "step %d %s: %s" % (step, k, describe_diff(got, batch[k]))
