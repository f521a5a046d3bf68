"""The library at the smallest legal grids and at strongly non-cubic ones, against the oracle, which
test_oracle_edge_sizes.py pins on the compiled reference at exactly these inputs (edge_cases.fields).

Every grid of edge_cases.CASES runs:
  * all six advection methods, scalar (both sampleOutsideFluid settings) and velocity, in place and out of place,
    at traces of 0.2 to 20 cells; on 3-D grids (nb = 1 and 2) also under tile modes 0, 1, 2 and automatic: bit for
    bit;
  * every point-wise operator, emptyDomain, flagsToOccupancy, rectangularBlur, signedDistanceField, upsampling and
    the backward operators: bit for bit;
  * the Jacobi solve at pTol = 0 with 1, 2, 3, 7 and 40 sweeps and at pTol > 0: p bit for bit, same iterations;
  * the PCG solve with each preconditioner: the tolerances of test_gpu_pcg.py, size-1 components exactly 0.
STEP_SHAPES also run the whole step (the fused convnet step at nb = 1 and 2, the operator path at nb = 2, Jacobi), 2-D
grids the fp32-model step, and 4x3x3 a step-graph replay.

Every array the library reads or writes is a 16-byte-aligned view into a buffer with a guard band of at least one
plane on each side, filled with a quiet-NaN sentinel: a kernel that reads past a small grid poisons its result, and
one that writes past it changes the sentinel, which is checked after every call, with trace_faults() == 0.

Which kernel a call reaches is proven, not assumed: a forced tile mode falls back to the two-kernel advection when
the tile kernel refuses a grid, so the launch count of every tile-mode call is compared with the same call under
tile mode 0 (the tile counts one launch, the two-kernel version two); a fixed-count Jacobi solve counts four
launches where the resident kernel runs its first maxIter - 1 sweeps and maxIter + 2 otherwise.  branches()
restates the dispatch predicates on the host, and test_table_reaches_every_branch (no GPU) keeps the table
reaching each of them.  A grid that cannot take a path says why in ROWS."""
import ctypes as C

import numpy as np
import pytest
import torch

import edge_cases
import oracle
from cases import bits_equal, describe_diff
from edge_cases import CASES, CASE_IDS, DT, STRENGTH
from fluidnet_b200 import synth
from step_cases import (Guards, MODE_TOL, OPS_TOL, case, close_per_entry, ctx, fill, make_batch, plane_of, quad_dims,
                        run, same_zero_bits, set_tile_mode, takes_fused_path)

METHODS = list(oracle.ADVECT_METHODS)
OURS_VEL = {"maccormackOurs", "rk2Ours", "rk3Ours"}       # advectVel methods the tile kernel runs
# Step states carry a density and no BCs: createPlumeBCs indexes past a 3-cell extent.
STEP_SHAPES = [(3, 3, 3), (4, 3, 3), (36, 3, 3), (4, 3, 300), (1028, 3, 3)]

# What each grid (nx, ny, nz) reaches, and why it cannot take a path it does not.
ROWS = {
    (3, 3, 3): "per-voxel kernels only, one interior cell (size-1 PCG component); no tile, quad or iter4: nx % 4 != 0",
    (4, 3, 3): "tile kernel smaller than one tile (nb = 1 and 2: the batch-wide tiles), quad bx = 1 with a 128-row y "
               "block on 3 rows",
    (4, 3, 5): "tile with an odd nz; jacobi iter4",
    (33, 3, 3): "per-voxel kernels (nx % 4 != 0)",
    (3, 17, 4): "per-voxel kernels (nx % 4 != 0), ny odd",
    (36, 3, 3): "tile: a last x tile of 4 cells; per-voxel step kernels (9 quads: not a power of two below 32)",
    (4, 17, 4): "tile: y spans three tiles",
    (1028, 3, 3): "long row: 9 quad blocks of bx = 32, the last one partial; 33 x tiles",
    (4, 300, 3): "tall (getDx from y): 38 y tiles",
    (4, 3, 300): "deep (getDx from z): 38 z tiles; the step with quad bx = 1 and 150 z blocks",
    (128, 8, 4): "k_jacobi_resident<4> with 1 block: three of the CTA's four groups idle",
    (128, 8, 5): "k_jacobi_resident<4> with 2 blocks, the second a partial z chunk",
    (128, 24, 4): "k_jacobi_resident<4> with 3 blocks",
    (256, 8, 4): "k_jacobi_resident<4> with 2 x blocks",
    (128, 8, 8): "k_jacobi_march at its smallest depth (1 and 2 sweeps; more run resident)",
    (3, 3, 1): "2-D per-voxel kernels, one interior cell",
    (5, 3, 1): "2-D: a 3-cell line (PCG without preconditioner)",
    (3, 41, 1): "2-D per-voxel kernels, tall",
    (4, 3, 1): "2-D k_jacobi_iter4 with one quad per row",
    (1028, 3, 1): "2-D long row, k_jacobi_iter4",
    (3, 600, 1): "2-D per-voxel kernels, very tall",
}


# ---------------------------------------------------------------------------------------------------------------
# Dispatch predicates, restated from the library
# ---------------------------------------------------------------------------------------------------------------
def tile_kernel(shape, nb):
    """launch_advect_vel_tile / launch_advect_scalar_tile (tfl_advect_tile.cu) accept the grid (16-byte-aligned
    views, whole grid on one GPU), at any nb: the nb ceil(nz / 8) z tiles of a batch stay within CUDA's 65535 blocks
    along gridDim.z wherever the grid check (check_launch_grid, nb nz <= 2 x 65535) lets the grid in."""
    nx, ny, nz = shape
    return nz > 1 and nx % 4 == 0 and nz >= 3


def tile_modes(shape, nb):
    """The tfl_debug_advect_tile modes test_advection forces (None: automatic): all of them on every 3-D grid."""
    return (None, 0, 1, 2) if shape[2] > 1 else (None,)


# (nb, conv mode) of test_step_fused_and_ops: the fused step alone and batched, and the operator path batched (an fp32
# model: fused_step_applies needs a tensor-core mode).
STEP_LEGS = ((1, "tf32x3"), (2, "tf32x3"), (2, "fp32"))


def resident_blocks(shape, nb):
    """Blocks (128 x 8 x 4 cells) of k_jacobi_resident<4> in the whole-grid solve, 0 where it refuses the grid.
    It runs for pTol == 0 and maxIter > 2 (tfl_solve_linear_system_jacobi, through launch_jacobi_block)."""
    nx, ny, nz = shape
    if nz == 1 or nx % 128 or ny % 8 or nz < 4 or nx * ny * nz * nb > (3 << 20):
        return 0
    return (nx // 128) * (ny // 8) * ((nz + 3) // 4) * nb


def jacobi_sweep_kernel(shape, nb):
    """The kernel launch_jacobi_iter picks for one sweep."""
    nx, ny, nz = shape
    big = nx * ny * nz * nb >= (4 << 20) or nz < 16
    if nz > 1 and big and nx % 128 == 0 and ny % 8 == 0 and nz >= 8:
        return "march"
    return "iter4" if nx % 4 == 0 else "iter"


def branches(shape):
    nx, ny, nz = shape
    out = set()
    if tile_kernel(shape, 1):
        out.add("tile")
        if nx % 32:
            out.add("tile-partial-x")
        if (ny + 7) // 8 >= 3:
            out.add("tile-multi-y")
        if nx < 32 and ny < 8 and nz < 8:
            out.add("tile-smaller-than-box")
    if nz > 1:
        out.add("two-kernel")          # tile mode 0 on every 3-D grid
    k = jacobi_sweep_kernel(shape, 1)
    out.add("jacobi-%s%s" % (k, "-2d" if nz == 1 else ""))
    for nb in edge_cases.batches(shape):
        blocks = resident_blocks(shape, nb)
        if blocks:
            out.add("resident-%d" % blocks)
            if blocks % 4:
                out.add("resident-idle-groups")
            if nz % 4:
                out.add("resident-partial-z")
            if nx // 128 > 1:
                out.add("resident-2x")
    interior = (nx - 2) * (ny - 2) * (nz - 2 if nz > 1 else 1)
    if interior == 1:
        out.add("pcg-size1")
    elif interior <= 4:
        out.add("pcg-small")
    if shape in STEP_SHAPES:
        q = quad_dims(1, nz, ny, nx)
        if q is None:
            out.add("step-scalar")
        else:
            (gx, gy, _), (bx, by, _) = q
            out.add("quad-bx%d" % bx)
            if gx * bx * 4 > nx:
                out.add("quad-partial-x")
            if gy * by > ny:
                out.add("quad-partial-y")
    return out


def test_table_reaches_every_branch():
    """No GPU: the grids keep reaching every dispatch branch named here, and ROWS describes each grid."""
    assert set(ROWS) == set(edge_cases.GRIDS)
    assert set(STEP_SHAPES) <= set(edge_cases.GRIDS)
    reached = set()
    for shape in edge_cases.GRIDS:
        reached |= branches(shape)
    want = {"tile", "tile-partial-x", "tile-multi-y", "tile-smaller-than-box", "two-kernel",
            "jacobi-march", "jacobi-iter4", "jacobi-iter", "jacobi-iter4-2d", "jacobi-iter-2d",
            "resident-1", "resident-2", "resident-3", "resident-idle-groups", "resident-partial-z", "resident-2x",
            "pcg-size1", "pcg-small", "step-scalar", "quad-bx1", "quad-bx32", "quad-partial-x", "quad-partial-y"}
    assert want <= reached, sorted(want - reached)
    assert resident_blocks((128, 8, 8), 1) and jacobi_sweep_kernel((128, 8, 8), 1) == "march"
    assert quad_dims(1, 3, 3, 4)[1] == (1, 128, 2)            # bx = 1, 128 rows per block on a 3-row grid
    assert quad_dims(1, 3, 3, 1028)[0][0] == 9
    # forced tile modes on the batch-wide tiles (nb = 2), and the step legs: fused at nb = 1 and 2, the operator path
    # at nb = 2
    assert any(nb == 2 and tile_kernel(s, nb) and {0, 1, 2} <= set(tile_modes(s, nb)) for s, nb in CASES)
    legs = {(nb, takes_fused_path({"mode": m, "nb": nb, "pbc": False})) for nb, m in STEP_LEGS}
    assert {(1, True), (2, True), (2, False)} <= legs, legs


# ---------------------------------------------------------------------------------------------------------------
# Guarded device copies
# ---------------------------------------------------------------------------------------------------------------


# ---------------------------------------------------------------------------------------------------------------
# Operators
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("shape,nb", CASES, ids=CASE_IDS)
def test_advection(orc, shape, nb):
    from fluidnet_b200 import tfluids
    is3d = shape[2] > 1
    modes = tile_modes(shape, nb)
    tile = tile_kernel(shape, nb)
    try:
        for trace in edge_cases.traces(shape):
            fl, U, s, _ = edge_cases.fields(shape, nb, trace)
            orc.setWallBcsForward(U, fl)
            pl = plane_of(fl)
            for method in METHODS:
                want_s = {o: orc.advectScalar(DT, s, U, fl, method, o, STRENGTH) for o in (False, True)}
                want_u = orc.advectVel(DT, U, fl, method, STRENGTH)
                counts = {}
                for mode in modes:
                    set_tile_mode(mode)
                    tag = "trace %g %s tile %s" % (trace, method, mode)
                    for o in (False, True):
                        (_, _, _, got), _, n_out = run(
                            "advectScalar " + tag, pl,
                            lambda ts, tu, tf, d: tfluids.advectScalar(DT, ts, tu, tf, method, d, o, STRENGTH),
                            s, U, fl, fill(s.shape))
                        assert bits_equal(got, want_s[o]), "%s outside %s: %s" % (tag, o, describe_diff(got, want_s[o]))
                        (got, _, _), _, n_in = run(
                            "advectScalar in place " + tag, pl,
                            lambda ts, tu, tf: tfluids.advectScalar(DT, ts, tu, tf, method, None, o, STRENGTH),
                            s, U, fl)
                        assert bits_equal(got, want_s[o]), "in place %s: %s" % (tag, describe_diff(got, want_s[o]))
                        counts[("s", o, mode)] = (n_out, n_in)
                    (_, _, got), _, n_out = run(
                        "advectVel " + tag, pl,
                        lambda tu, tf, d: tfluids.advectVel(DT, tu, tf, method, d, STRENGTH), U, fl, fill(U.shape))
                    assert bits_equal(got, want_u), "advectVel %s: %s" % (tag, describe_diff(got, want_u))
                    (got, _), _, n_in = run(
                        "advectVel in place " + tag, pl,
                        lambda tu, tf: tfluids.advectVel(DT, tu, tf, method, None, STRENGTH), U, fl)
                    assert bits_equal(got, want_u), "advectVel in place %s: %s" % (tag, describe_diff(got, want_u))
                    counts[("u", None, mode)] = (n_out, n_in)
                for mode in (1, 2):
                    if mode not in modes:
                        continue
                    for o in (False, True):
                        saved = 1 if tile and method == "maccormackOurs" else 0
                        assert counts[("s", o, mode)] == tuple(n - saved for n in counts[("s", o, 0)]), \
                            ("advectScalar launches", shape, method, mode, counts)
                    saved = 1 if tile and method in OURS_VEL else 0
                    assert counts[("u", None, mode)] == tuple(n - saved for n in counts[("u", None, 0)]), \
                        ("advectVel launches", shape, method, mode, counts)
    finally:
        set_tile_mode(None)


@pytest.mark.gpu
@pytest.mark.parametrize("shape,nb", CASES, ids=CASE_IDS)
def test_operators(orc, shape, nb):
    from fluidnet_b200 import tfluids
    is3d = shape[2] > 1
    fl, U, s, p = edge_cases.fields(shape, nb)
    orc.setWallBcsForward(U, fl)
    pl = plane_of(fl)
    gpu_ops = {
        "setWallBcs": lambda u, f, ts, tp: tfluids.setWallBcsForward(u, f),
        "velocityUpdate": lambda u, f, ts, tp: tfluids.velocityUpdateForward(u, f, tp),
        "addBuoyancy": lambda u, f, ts, tp: tfluids.addBuoyancy(u, f, ts, edge_cases.GRAVITY, 0.1),
        "addGravity": lambda u, f, ts, tp: tfluids.addGravity(u, f, edge_cases.GRAVITY, 0.1),
        "vorticityConfinement": lambda u, f, ts, tp: tfluids.vorticityConfinement(u, f, 0.4),
    }
    for name, fn in edge_cases.pointwise_ops(fl, s, p):
        want = U.copy()
        fn(orc, want)
        (got, _, _, _), _, _ = run(name, pl, gpu_ops[name], U, fl, s, p)
        assert bits_equal(got, want), "%s %s" % (name, describe_diff(got, want))
    # setWallBcs as a mask multiply (tfluids.SetWallBcs)
    want = U.copy()
    orc.setWallBcsForward(want, fl, True)
    (mask, _), _, _ = run("setWallBcs mask", pl, lambda m, f: tfluids.setWallBcsForward(m, f), np.ones_like(U), fl)
    assert bits_equal(U * mask, want)
    want = orc.velocityDivergenceForward(U, fl)
    (_, _, got), _, _ = run("divergence", pl, lambda u, f, d: tfluids.velocityDivergenceForward(u, f, d),
                            U, fl, fill(fl.shape))
    assert bits_equal(got, want), "divergence " + describe_diff(got, want)
    inv = (p > 0).astype(np.float32)
    want = s.copy()
    orc.applyBC(want, inv, p)
    (got, _, _), _, _ = run("applyBC", pl, tfluids.applyBC, s, inv, p)
    assert bits_equal(got, want), "applyBC " + describe_diff(got, want)
    big = (U * np.float32(1e6)).astype(np.float32)
    want = big.copy()
    orc.clamp(want, -1e6, 1e6)
    (got,), _, _ = run("clamp", pl, lambda x: tfluids.clamp(x, -1e6, 1e6), big)
    assert bits_equal(got, want), "clamp " + describe_diff(got, want)
    for bnd in (1, 2):
        want = orc.emptyDomain(np.zeros_like(fl), is3d, bnd)
        if bnd in edge_cases.empty_domain_bnds(shape):
            (got,), _, _ = run("emptyDomain %d" % bnd, pl, lambda f: tfluids.emptyDomain(f, is3d, bnd),
                               np.zeros_like(fl))
            assert bits_equal(got, want), "emptyDomain %d" % bnd
        else:
            with pytest.raises(AssertionError, match="not big enough"):
                run("emptyDomain %d" % bnd, pl, lambda f: tfluids.emptyDomain(f, is3d, bnd), np.zeros_like(fl))
    (_, got), _, _ = run("flagsToOccupancy", pl, tfluids.flagsToOccupancy, fl, fill(fl.shape, 55.0))
    assert bits_equal(got, orc.flagsToOccupancy(fl))
    for rad in edge_cases.blur_radii(shape):
        want = orc.rectangularBlur(U, rad, is3d)
        (src, got), _, _ = run("blur %d" % rad, pl, lambda a, d: tfluids.rectangularBlur(a, rad, is3d, d),
                               U, fill(U.shape))
        assert bits_equal(got, want), "blur %d %s" % (rad, describe_diff(got, want))
        assert bits_equal(src, U), "rectangularBlur modified its input"
    for rad in (1, 3):
        (_, got), _, _ = run("sdf %d" % rad, pl, lambda f, d: tfluids.signedDistanceField(f, rad, is3d, d),
                             fl, fill(fl.shape))
        assert bits_equal(got, orc.signedDistanceField(fl, rad, is3d)), "signedDistanceField %d" % rad
    for ratio in edge_cases.UP_RATIOS:
        up = orc.volumetricUpSamplingNearestForward(ratio, U)
        (_, got), _, _ = run("upsample %d" % ratio, pl,
                             lambda x, o: tfluids.volumetricUpSamplingNearestForward(ratio, x, o), U, fill(up.shape))
        assert bits_equal(got, up), "upsampling %d" % ratio
        g = (up * np.float32(0.5) - np.float32(0.25)).astype(np.float32)
        (_, _, got), _, _ = run("upsample backward %d" % ratio, pl,
                                lambda x, go, gi: tfluids.volumetricUpSamplingNearestBackward(ratio, x, go, gi),
                                U, g, fill(U.shape))
        assert bits_equal(got, orc.volumetricUpSamplingNearestBackward(ratio, U, g)), "upsampling backward"
    want = orc.velocityDivergenceBackward(U, fl, p)
    (_, _, _, got), _, _ = run("divergence backward", pl, tfluids.velocityDivergenceBackward, U, fl, p, fill(U.shape))
    assert bits_equal(got, want), "velocityDivergenceBackward " + describe_diff(got, want)
    want = orc.velocityUpdateBackward(U, fl, p, U)
    (_, _, _, _, got), _, _ = run("update backward", pl, tfluids.velocityUpdateBackward, U, fl, p, U, fill(fl.shape))
    assert bits_equal(got, want), "velocityUpdateBackward " + describe_diff(got, want)


@pytest.mark.gpu
@pytest.mark.parametrize("shape,nb", CASES, ids=CASE_IDS)
def test_jacobi(orc, shape, nb):
    from fluidnet_b200 import tfluids
    is3d = shape[2] > 1
    fl, U, _, _ = edge_cases.fields(shape, nb)
    orc.setWallBcsForward(U, fl)
    div = orc.velocityDivergenceForward(U, fl)
    blocks = resident_blocks(shape, nb)
    for ptol, iters in ((0.0, 1), (0.0, 2), (0.0, 3), (0.0, 7), (0.0, 40), (1e-3, 500)):
        want = fill(div.shape, 9.0)
        rw = orc.solveLinearSystemJacobi(want, fl, div, is3d, ptol, iters)
        (got, _, _), rg, launches = run("jacobi %g %d" % (ptol, iters), plane_of(fl),
                                        lambda tp, f, d: tfluids.solveLinearSystemJacobi(tp, f, d, is3d, ptol, iters),
                                        fill(div.shape, 9.0), fl, div)
        what = "jacobi pTol %g maxIter %d" % (ptol, iters)
        assert bits_equal(got, want), "%s: %s" % (what, describe_diff(got, want))
        assert abs(rg - rw) <= 1e-5 * max(abs(rw), 1e-12) + 1e-12, (what, rg, rw)
        assert tfluids.solveLinearSystemJacobi.last_iterations == orc.last_jacobi_iters, what
        if ptol == 0.0:
            resident = blocks > 0 and iters > 2
            assert launches == (4 if resident else iters + 2), (what, "resident" if resident else "per sweep", launches)


@pytest.mark.gpu
@pytest.mark.parametrize("shape,nb", CASES, ids=CASE_IDS)
def test_pcg(orc, shape, nb):
    from fluidnet_b200 import tfluids
    is3d = shape[2] > 1
    fl, U, _, _ = edge_cases.fields(shape, nb)
    orc.setWallBcsForward(U, fl)
    div = orc.velocityDivergenceForward(U, fl)
    tol, max_iter = 1e-5, 3000     # unpreconditioned CG needs about n iterations on the 1026-cell lines
    single = np.zeros(fl.shape, bool)          # cells of size-1 components
    for b in range(nb):
        comp, sizes = orc.findConnectedFluidComponents(fl, is3d, b)
        for ic, size in enumerate(sizes):
            if size == 1:
                single[b, 0][comp == ic] = True
    for precond in ("none", "ilu0", "ic0"):
        want = np.zeros(fl.shape, np.float32)
        rw = orc.solveLinearSystemPCG(want, fl, div, is3d, tol, max_iter, precond)
        start = np.random.default_rng(3).random(fl.shape).astype(np.float32)      # must be overwritten
        (got, _, _), rg, _ = run("pcg " + precond, plane_of(fl),
                                 lambda tp, f, d: tfluids.solveLinearSystemPCG(tp, f, d, is3d, tol, max_iter, precond),
                                 start, fl, div)
        assert rg < 2 * tol and rw < 2 * tol, (precond, rg, rw)
        assert abs(tfluids.solveLinearSystemPCG.last_iterations - orc.last_pcg_iters) <= 2, precond
        assert not np.isnan(got).any()
        assert np.all(got[fl != 1] == 0)
        assert np.all(got[single].view(np.uint32) == 0), "%s: a size-1 component is not exactly +0" % precond
        assert np.abs(got - want).max() <= 2e-3 * np.abs(want).max(), precond


# ---------------------------------------------------------------------------------------------------------------
# The whole step
# ---------------------------------------------------------------------------------------------------------------
def guarded_batch(batch, gd):
    return {k: gd.put(v) for k, v in batch.items()}


def host(b):
    return {k: v.cpu().numpy() for k, v in b.items()}


def step_checks(gd, what):
    torch.cuda.synchronize()
    gd.check(what)
    assert ctx().trace_faults() == 0, what


@pytest.mark.gpu
@pytest.mark.parametrize("shape", STEP_SHAPES, ids=["%dx%dx%d" % s for s in STEP_SHAPES])
def test_step_fused_and_ops(orc, shape):
    """tfl_simulate_step on each of STEP_LEGS (the fused convnet path at nb = 1 and 2, the operator path at nb = 2),
    two steps each, against the oracle (density bit for bit, U and p within MODE_TOL) and against the operator
    sequence (within OPS_TOL with the same zeros)."""
    from fluidnet_b200 import simulate
    from fluidnet_b200.model import ProjectionModel
    nx, ny, nz = shape
    mnp = synth.make_model(True)
    for nb, mode in STEP_LEGS:
        gm = ProjectionModel.from_model(mnp)
        gm.set_mode(mode)
        c = case((nz, ny, nx), nb=nb, flags="empty", state="density", mode=mode)
        batch = make_batch(orc, c)
        gd = Guards(nx * ny)
        fused, ops = guarded_batch(batch, gd), guarded_batch(batch, gd)
        ctx().trace_faults()
        for step in range(2):
            ref = host(fused)
            for k in ops:
                ops[k].copy_(fused[k])
            oracle.simulate(orc, c["mconf"], ref, mnp)
            simulate.simulate_fused(None, c["mconf"], fused, gm)
            simulate.simulate(None, c["mconf"], ops, gm)
            what = "%s nb %d %s step %d" % (shape, nb, mode, step)
            step_checks(gd, what)
            got, opg = host(fused), host(ops)
            assert bits_equal(got["density"], ref["density"]), \
                "%s density: %s" % (what, describe_diff(got["density"], ref["density"]))
            for k in ("UDiv", "pDiv"):
                close_per_entry(got[k], ref[k], MODE_TOL[mode], "%s %s vs oracle" % (what, k))
                close_per_entry(got[k], opg[k], OPS_TOL, "%s %s vs ops" % (what, k))
                assert same_zero_bits(got[k], opg[k]), "%s %s zeros" % (what, k)
        assert orc.trace_faults() == 0


@pytest.mark.gpu
@pytest.mark.parametrize("shape", STEP_SHAPES, ids=["%dx%dx%d" % s for s in STEP_SHAPES])
def test_step_jacobi(orc, shape):
    """The Jacobi step (no network): bit for bit against the oracle."""
    from fluidnet_b200 import simulate
    nx, ny, nz = shape
    c = case((nz, ny, nx), flags="empty", state="density")
    batch = make_batch(orc, c)
    mconf = dict(c["mconf"], simMethod="jacobi", maxIter=12)
    gd = Guards(nx * ny)
    batch["div"] = np.zeros_like(batch["pDiv"])
    gb = guarded_batch(batch, gd)
    del batch["div"]
    for step in range(2):
        simulate.simulate_fused(None, mconf, gb, None)
        oracle.simulate(orc, mconf, batch, None)
        step_checks(gd, "jacobi step %d" % step)
        for k in ("density", "UDiv", "pDiv"):
            got = gb[k].cpu().numpy()
            assert bits_equal(got, batch[k]), "step %d %s: %s" % (step, k, describe_diff(got, batch[k]))


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(3, 3), (3, 41)], ids=["3x3", "3x41"])
def test_step_2d_fp32_model(orc, shape):
    from fluidnet_b200 import simulate
    from fluidnet_b200.model import ProjectionModel
    nx, ny = shape
    flags = synth.make_flags(nx, ny, 1, False)
    U = synth.make_smooth_velocity(flags, False, amp=3.0)
    orc.setWallBcsForward(U, flags)
    batch = {"pDiv": np.zeros_like(flags), "UDiv": U, "flags": flags, "density": synth.make_density(flags)}
    mnp = synth.make_model(False)
    gm = ProjectionModel.from_model(mnp)
    mconf = oracle.default_mconf(dt=0.1, maccormackStrength=0.6, buoyancyScale=1.0, vorticityConfinementAmp=0.0,
                                 simMethod="convnet", is3D=False)
    gd = Guards(nx * ny)
    gb = guarded_batch(batch, gd)
    for step in range(2):
        simulate.simulate_fused(None, mconf, gb, gm)
        oracle.simulate(orc, mconf, batch, mnp)
        step_checks(gd, "2-D step %d" % step)
        got = host(gb)
        assert bits_equal(got["density"], batch["density"]), describe_diff(got["density"], batch["density"])
        for k in ("UDiv", "pDiv"):
            close_per_entry(got[k], batch[k], MODE_TOL["fp32"], "2-D step %d %s" % (step, k))
        for k in batch:
            gb[k].copy_(torch.from_numpy(batch[k]))         # next step from the oracle's state


@pytest.mark.gpu
def test_step_graph_replay_on_a_tiny_grid(orc):
    """A step graph captured at 4x3x3 replays the direct step bit for bit."""
    from fluidnet_b200 import simulate
    from fluidnet_b200.model import ProjectionModel
    c = case((3, 3, 4), flags="empty", state="density")
    batch = make_batch(orc, c)
    gm = ProjectionModel.from_model(synth.make_model(True))
    gd = Guards(12)
    ga, gb = guarded_batch(batch, gd), guarded_batch(batch, gd)
    stream = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(stream):
        simulate.simulate_fused(None, c["mconf"], ga, gm)
        simulate.simulate_fused(None, c["mconf"], gb, gm)
        graph = simulate.StepGraph(c["mconf"], gb, gm)
        try:
            for replay in range(3):
                graph.launch()
                simulate.simulate_fused(None, c["mconf"], ga, gm)
                stream.synchronize()
                for k in ("density", "UDiv", "pDiv"):
                    assert torch.equal(ga[k].view(torch.int32), gb[k].view(torch.int32)), (replay, k)
        finally:
            graph.close()
    step_checks(gd, "graph")


# ---------------------------------------------------------------------------------------------------------------
# The grid bound
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_grid_bound_keeps_block_offsets_in_32_bits():
    """make_geo refuses n >= 2^31 cells per (batch, channel) block, which cell() indexes in 32 bits; per-block
    offsets only, so a batch of two 1024^3 grids is accepted.  Only the descriptor is checked (no launch)."""
    from fluidnet_b200._lib import Grid
    c = ctx()
    c.lib.tfl_debug_make_geo.argtypes = [C.c_void_p, C.POINTER(Grid), C.c_int]

    def geo(nb, n):
        g = Grid(C.c_void_p(256), nb, 1, n, n, n)
        return c.lib.tfl_debug_make_geo(c.h, C.byref(g), 1)

    assert geo(1, 1291) == 1
    assert "grid too large" in c.lib.tfl_last_error(c.h).decode()
    assert geo(1, 1290) == 0
    assert geo(2, 1024) == 0
