"""advectVel('maccormackOurs') over shared-memory tiles (tfl_advect_tile.cu) against the CPU oracle, bit for
bit, in every configuration the dispatcher can choose: the two-kernel version (mode 0), the tile kernel with
a forward halo of 1 and of 2 cells, and velocities whose traces stay inside the halo
(amp 2: 0.2 cell), leave halo 1 (amp 8), and leave every halo (amp 25: the backward pass re-evaluates the
forward values it needs).  Grids: not multiples of the tile, with solids (sphere + slab), with the exotic
flag mix (empty / outflow / stick cells), and one plane thinner than a tile."""
import ctypes as C

import numpy as np
import pytest

from cases import bits_equal, describe_diff
from fluidnet_b200 import synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gpu():
    from gpu_backend import GpuBackend
    return GpuBackend()


def set_tile(mode):
    from fluidnet_b200 import tfluids
    ctx = tfluids.context()
    ctx.lib.tfl_debug_advect_tile.argtypes = [C.c_void_p, C.c_int]
    assert ctx.lib.tfl_debug_advect_tile(ctx.h, mode) == 0


GRIDS = [((40, 24, 20), True, False), ((36, 20, 12), True, True), ((64, 16, 5), False, False)]


@pytest.mark.parametrize("dims,geom,exotic", GRIDS, ids=["40x24x20_geom", "36x20x12_exotic", "64x16x5_empty"])
@pytest.mark.parametrize("amp", [2.0, 8.0, 25.0])
def test_tile_modes_match_oracle(orc, gpu, dims, geom, exotic, amp):
    nx, ny, nz = dims
    flags = synth.make_flags(nx, ny, nz, True, nb=1, geometry=geom, exotic=exotic)
    U = synth.make_velocity(flags, True, amp=amp)
    orc.setWallBcsForward(U, flags)
    want = orc.advectVel(0.1, U, flags, "maccormackOurs", 0.6)
    try:
        for mode in (0, 1, 2, -1):
            set_tile(mode)
            got = gpu.advectVel(0.1, U, flags, "maccormackOurs", 0.6)
            assert bits_equal(got, want), "mode %d: %s" % (mode, describe_diff(got, want))
            got = gpu.advectVel(0.1, U, flags, "maccormackOurs", 0.6, in_place=True)
            assert bits_equal(got, want), "in place, mode %d: %s" % (mode, describe_diff(got, want))
    finally:
        set_tile(-1)
    assert gpu.trace_faults() == 0


@pytest.mark.parametrize("dims,geom,exotic", GRIDS, ids=["40x24x20_geom", "36x20x12_exotic", "64x16x5_empty"])
@pytest.mark.parametrize("amp", [2.0, 8.0, 25.0])
def test_scalar_tile_modes_match_oracle(orc, gpu, dims, geom, exotic, amp):
    """advectScalar('maccormackOurs') on the tiles, both sampleOutsideFluid settings, every dispatcher choice."""
    nx, ny, nz = dims
    flags = synth.make_flags(nx, ny, nz, True, nb=1, geometry=geom, exotic=exotic)
    U = synth.make_velocity(flags, True, amp=amp)
    orc.setWallBcsForward(U, flags)
    rho = synth.make_density(flags)
    rho[np.random.RandomState(3).rand(*rho.shape) < 0.3] = 0.0          # zero bounds in the clamp
    try:
        for outside in (False, True):
            want = orc.advectScalar(0.1, rho, U, flags, "maccormackOurs", outside, 0.6)
            for mode in (0, 1, 2, -1):
                set_tile(mode)
                got = gpu.advectScalar(0.1, rho, U, flags, "maccormackOurs", outside, 0.6)
                assert bits_equal(got, want), "outside %s mode %d: %s" % (outside, mode, describe_diff(got, want))
            got = gpu.advectScalar(0.1, rho, U, flags, "maccormackOurs", outside, 0.6, in_place=True)
            assert bits_equal(got, want), "in place: " + describe_diff(got, want)
    finally:
        set_tile(-1)
    assert gpu.trace_faults() == 0


def test_zero_bounds_keep_their_sign(orc, gpu):
    """The clamp's min / max run on FMNMX with an exact re-evaluation when a bound is +-0: fields with large
    regions of +0 and -0 velocities must still match the reference's compare-and-keep bit for bit."""
    nx, ny, nz = 40, 24, 20
    flags = synth.make_flags(nx, ny, nz, True, nb=1, geometry=True)
    U = synth.make_smooth_velocity(flags, True, amp=3.0)
    rng = np.random.RandomState(5)
    U[rng.rand(*U.shape) < 0.35] = 0.0
    U[rng.rand(*U.shape) < 0.2] = -0.0
    orc.setWallBcsForward(U, flags)
    want = orc.advectVel(0.1, U, flags, "maccormackOurs", 0.6)
    try:
        for mode in (1, 2):
            set_tile(mode)
            got = gpu.advectVel(0.1, U, flags, "maccormackOurs", 0.6)
            assert bits_equal(got, want), "mode %d: %s" % (mode, describe_diff(got, want))
    finally:
        set_tile(-1)


def test_halo_choice_follows_the_velocities(gpu):
    """The automatic mode reads the longest trace of earlier calls (asynchronously) and widens the halo or
    falls back to the two-kernel version; whatever it picks, results equal mode 0."""
    import torch
    from fluidnet_b200 import tfluids
    nx, ny, nz = 64, 32, 24
    flags = synth.make_flags(nx, ny, nz, True, nb=1, geometry=True)
    tf = torch.from_numpy(flags).cuda()
    try:
        for amp in (2.0, 9.0, 30.0, 2.0):
            U = torch.from_numpy(synth.make_velocity(flags, True, amp=amp)).cuda()
            tfluids.setWallBcsForward(U, tf)
            set_tile(0)
            ref = torch.empty_like(U)
            tfluids.advectVel(0.1, U, tf, "maccormackOurs", ref, 0.6)
            set_tile(-1)
            for _ in range(3):                   # the choice may change between these calls
                out = torch.empty_like(U)
                tfluids.advectVel(0.1, U, tf, "maccormackOurs", out, 0.6)
                torch.cuda.synchronize()
                assert torch.equal(out.view(torch.int32), ref.view(torch.int32)), "amp %g" % amp
    finally:
        set_tile(-1)
