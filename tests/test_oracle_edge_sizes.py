"""Smallest legal grids and strongly non-cubic ones (the reference's own tests sweep odd sizes,
tfluids/test_tfluids.lua): the oracle against the compiled reference, bit for bit, on 3-cell domains (a
single interior cell), thin slabs and long rows, for every advection method and every point-wise operator.
CPU only; the GPU parity tests compare against this oracle."""
import numpy as np
import pytest

import oracle
from oracle import api
import ref_record
from cases import bits_equal, describe_diff
from fluidnet_b200 import synth

SHAPES = [((3, 3, 3), True), ((4, 3, 5), True), ((33, 3, 3), True), ((3, 17, 4), True),
          ((3, 3, 1), False), ((5, 3, 1), False), ((3, 41, 1), False)]
IDS = ["%dx%dx%d-%s" % (s + ("3d" if d else "2d",)) for s, d in SHAPES]
METHODS = list(oracle.ADVECT_METHODS)


@pytest.fixture(scope="module")
def ref():
    return ref_record.reference()


def fields(shape, is3d, seed):
    nx, ny, nz = shape
    rng = np.random.default_rng(seed)
    fl = synth.make_flags(nx, ny, nz, is3d, nb=2, geometry=False)
    U = (rng.standard_normal((2, 3 if is3d else 2, nz, ny, nx)) * 1.5).astype(np.float32)
    s = rng.random(fl.shape).astype(np.float32)
    return fl, U, s


@pytest.mark.parametrize("shape,is3d", SHAPES, ids=IDS)
def test_advection_on_tiny_grids(orc, ref, shape, is3d):
    fl, U, s = fields(shape, is3d, 1)
    orc.setWallBcsForward(U, fl)
    for method in METHODS:
        for outside in (False, True):
            a, b = orc.advectScalar(0.3, s, U, fl, method, outside, 0.75), ref.advectScalar(0.3, s, U, fl, method, outside, 0.75)
            assert bits_equal(a, b), "advectScalar %s %s" % (method, describe_diff(a, b))
        a, b = orc.advectVel(0.3, U, fl, method, 0.75), ref.advectVel(0.3, U, fl, method, 0.75)
        assert bits_equal(a, b), "advectVel %s %s" % (method, describe_diff(a, b))


@pytest.mark.parametrize("shape,is3d", SHAPES, ids=IDS)
def test_pointwise_on_tiny_grids(orc, ref, shape, is3d):
    fl, U, s = fields(shape, is3d, 2)
    p = (s - np.float32(0.5)).astype(np.float32)
    for name, fn in (
        ("setWallBcs", lambda be, u: be.setWallBcsForward(u, fl)),
        ("velocityUpdate", lambda be, u: be.velocityUpdateForward(u, fl, p)),
        ("addBuoyancy", lambda be, u: be.addBuoyancy(u, fl, s, [0.2, -0.5, 0.1], 0.1)),
        ("addGravity", lambda be, u: be.addGravity(u, fl, [0.2, -0.5, 0.1], 0.1)),
        ("vorticityConfinement", lambda be, u: be.vorticityConfinement(u, fl, 0.4)),
    ):
        a, b = U.copy(), U.copy()
        fn(orc, a)
        fn(ref, b)
        assert bits_equal(a, b), "%s %s" % (name, describe_diff(a, b))
    a, b = orc.velocityDivergenceForward(U, fl), ref.velocityDivergenceForward(U, fl)
    assert bits_equal(a, b), describe_diff(a, b)
    assert bits_equal(orc.flagsToOccupancy(fl), ref.flagsToOccupancy(fl))
    for rad in (1, 2):
        assert bits_equal(orc.signedDistanceField(fl, rad, is3d), ref.signedDistanceField(fl, rad, is3d))
        assert bits_equal(orc.rectangularBlur(U, rad, is3d), ref.rectangularBlur(U, rad, is3d))
    assert bits_equal(orc.velocityDivergenceBackward(U, fl, p), ref.velocityDivergenceBackward(U, fl, p))
