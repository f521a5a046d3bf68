"""The PCG solve (tfl_pcg.cu) against the float64 restatement of tests/pcg_reference.py.

(a) The preconditioner alone, through tfl_debug_pcg_precond (labelling, k_build, the FACTOR sweep and one solve
    sweep of tfl_solve_linear_system_pcg; z = M^-1 r in the natural layout).  Per voxel
        |z - z64| <= KAPPA * S,   S = M^-1 |r| in float64,
    and z is +0.0 bit for bit outside every system.  S is the natural scale: R is an M-matrix (positive diagonal,
    non-positive off-diagonal, the pivot guard keeps it so), hence R^-1 >= 0 and M^-1 = R^-1 R^-T >= 0 entrywise,
    |M^-1 r| <= S, and a rounding error made at any cell reaches cell i through the same non-negative weights that
    carry |r| into S_i.  Each cell's fp32 sweep makes 4 roundings forward, 3 backward, about 6 in its pivot (the
    ptxas order is restated in pcg_reference.emulate_sweep_fp32), each of relative size u = 2^-24 of a term that
    is itself at most the matching majorant.  Summed along the weighted dependency paths, whose weights decay by a
    factor of about sum pre^2 ~ 0.55 per wavefront in the interior (so the effective depth is tens of cells, not
    nx + ny + nz; along a 1-wide chain pre = 1 exactly and nothing is rounded in the factor), that gives
    |err| <~ (13 u) (1 + 0.55 + 0.55^2 + ...) * a few ~ 2^-19 S.  KAPPA = 2^-16 leaves a factor of 8 for the
    constants; test_sweep_emulation_within_kappa confirms it on the CPU (the fp32 emulation of the kernel's
    arithmetic stays below KAPPA / 8 on every case of the table), and shows that the emulation of an unmasked
    cross-CTA z- term (3- and 4-cell components across a chunk boundary: z = r_k + r_k-1 instead of r_k) does not.
(b) Fixed-count iterates through tfl_solve_linear_system_pcg: maxIter in {0, 1, 2, 4} (maxIter + 1 iterations) with
    a tol that only exactly solved components (a few cells) reach, per component |p - p64| <= TAU[k] max|p64|.
    TAU is calibrated on the CPU by the oracle's fp32 orc_pcg on the same cases (test_oracle_iterates_within_tau:
    at most TAU / 8).
(c) Components freeze independently: a tol picked on the float64 trajectories so that small components stop
    within a few iterations, some of them before their exact solve, while the large ones run all maxIter + 1;
    no component's rr comes within 2x of tol^2, and each component is held to its own iterate within TAU.

The CPU tests of this file run every case through the oracle and the fp32 emulation, so the bounds are fixed
without a GPU."""
import ctypes as C
import zlib

import numpy as np
import pytest

import pcg_reference as R

KAPPA = 2.0 ** -16
TAU = {0: 4e-6, 1: 8e-6, 2: 8e-6, 4: 1.6e-5}
MAX_GRID_PROBE = 4500                          # planes of the thin column (GP = 1): more chunks than CTAs


# ---------------------------------------------------------------------------------------------------------------
# Cases
# ---------------------------------------------------------------------------------------------------------------
def _carve(f, is3d, cells):
    """Fluid at `cells` ((k, j, i) tuples) inside an obstacle shell (6- or 4-neighbourhood)."""
    nb6 = ((0, 0, 1), (0, 0, -1), (0, 1, 0), (0, -1, 0)) + (((1, 0, 0), (-1, 0, 0)) if is3d else ())
    for k, j, i in cells:
        for dk, dj, di in nb6:
            if (k + dk, j + dj, i + di) not in cells:
                f[k + dk, j + dj, i + di] = 2
    for c in cells:
        f[c] = 1


def make_flags(orc, n, nb=1, is3d=True, seed=0, small=True, empty=False):
    """(nx, ny, nz) grid: obstacle border, 4 % random obstacles, a wall across y = ny / 2 (large components
    below and above), and in the upper half small components: vertical 2- to 5-cell columns (3-D) starting at
    every z, so that some cross any chunk boundary; a 1-cell-wide chain of 8 along x (pivot guard at its end);
    x-runs of 2 to 5 cells (2-D); strips along y of 3 and 6 cells one obstacle apart along x (several components
    in one warp's wavefront).  empty: a row of Empty (Dirichlet) cells."""
    nx, ny, nz = n
    rng = np.random.default_rng(seed)
    flags = np.ones((nb, 1, nz, ny, nx), np.float32)
    orc.emptyDomain(flags, is3d, 1)
    for b in range(nb):
        f = flags[b, 0]
        f[:, ny // 2, :] = 2
        f[rng.random(f.shape) < 0.04] = 2
        if empty:
            f[(slice(1, nz - 1) if is3d else slice(0, 1)), ny - 3, 2:nx - 2] = 4
        if not small:
            continue
        k0 = nz // 2 if is3d else 0
        y, x, t = ny // 2 + 2, 2, 0
        top = ny - (5 if empty else 3)
        shapes = []
        if is3d:
            shapes += [("col", L, z0) for z0 in range(1, 9) for L in (3, 4, 2, 5) if z0 + L <= nz - 1]
        else:
            shapes += [("run", L, 0) for L in (2, 3, 4, 5)] * 2
        shapes += [("run", 8, 0), ("strips", 3, 0), ("strips", 6, 0)]
        for kind, L, z0 in shapes:
            width = {"col": 1, "run": L, "strips": 7}[kind]
            height = {"col": 1, "run": 1, "strips": L}[kind]
            if x + width > nx - 2:
                x, y = 2, y + 3 + (3 if kind == "strips" else 0)
            if y + height > top or x + width > nx - 2:
                continue
            if kind == "col":
                _carve(f, is3d, {(z0 + d, y, x) for d in range(L)})
            elif kind == "run":
                _carve(f, is3d, {(k0, y, x + d) for d in range(L)})
            else:
                for s in range(0, 7, 2):
                    _carve(f, is3d, {(k0, y + d, x + s) for d in range(L)})
            x += width + 2
            t += 1
    tmp = flags.copy()
    orc.emptyDomain(tmp, is3d, 1)
    flags[tmp == 2] = 2
    return flags


def make_div(orc, flags, is3d, seed=0):
    rng = np.random.default_rng(seed + 100)
    nb, _, nz, ny, nx = flags.shape
    U = rng.standard_normal((nb, 3 if is3d else 2, nz, ny, nx)).astype(np.float32)
    orc.setWallBcsForward(U, flags)
    return orc.velocityDivergenceForward(U, flags)


# name: (nx, ny, nz), nb, is3d, forced planes per CTA (None: automatic), extra make_flags arguments
CASES = {
    "3d-nx>ny-gp1": ((20, 14, 12), 2, True, 1, {}),
    "3d-nx>ny-gp2": ((20, 14, 12), 2, True, 2, {}),
    "3d-nx>ny-gp3": ((20, 14, 12), 2, True, 3, {}),
    "3d-nx>ny-gp7": ((20, 14, 12), 2, True, 7, {}),
    "3d-nx>ny-auto": ((20, 14, 12), 2, True, None, {}),
    "3d-ny>nx-gp3": ((12, 20, 11), 2, True, 3, {}),
    "3d-ny>nx-gp7-empty": ((12, 20, 11), 1, True, 7, {"empty": True}),
    "3d-cube-gp2": ((16, 16, 16), 1, True, 2, {}),
    "3d-ny31-gp3": ((14, 31, 9), 1, True, 3, {}),
    "3d-ny32-gp2": ((12, 32, 9), 1, True, 2, {}),
    "3d-ny33-gp7": ((12, 33, 10), 2, True, 7, {}),
    "3d-ny64-auto": ((10, 64, 8), 1, True, None, {}),
    "3d-ny65-gp3": ((10, 65, 8), 1, True, 3, {}),
    "3d-ny128-gp1": ((9, 128, 7), 1, True, 1, {}),
    "2d-nb5-gp2": ((24, 20, 1), 5, False, 2, {}),
    "2d-ny>nx-auto": ((18, 40, 1), 3, False, None, {"empty": True}),
    "2d-ny960": ((8, 960, 1), 1, False, None, {}),
    "3d-column-multichunk": ((5, 5, MAX_GRID_PROBE), 1, True, 1, {"small": False}),
}
# fixed-count iterates: the cases above minus the largest
ITER_CASES = [k for k in CASES if k not in ("2d-ny960", "3d-column-multichunk")]


def crossing_small_components(sys, groups):
    """Sizes of the components of 2-4 cells with cells on both sides of a chunk boundary (planes pl = b nz + k,
    pl % groups == 0 starts a chunk)."""
    if not sys.is3d or not groups:
        return []
    pl = sys.batch * sys.shape[2] + sys.k
    sizes = []
    for c in np.flatnonzero(sys.size < 5):
        p = pl[sys.cid == c]
        if any(q % groups == 0 and (q - 1) in p for q in p):
            sizes.append(int(sys.size[c]))
    return sizes


_built = {}


def build_case(orc, name, precond="ic0"):
    """(flags, div, System) of a named case; the grid depends on the name alone (not on which cases were built
    before it), so every precond mode and every test selection sees the grid the CPU checks validated."""
    key = (name, precond)
    if key not in _built:
        n, nb, is3d, gp, kw = CASES[name]
        seed = zlib.crc32(name.encode())
        flags = make_flags(orc, n, nb, is3d, seed=seed, **kw)
        div = make_div(orc, flags, is3d, seed=seed)
        _built[key] = (flags, div, R.System(orc, flags, is3d, precond))
    return _built[key]


# ---------------------------------------------------------------------------------------------------------------
# CPU: the case table is valid, and the bounds are calibrated without a GPU
# ---------------------------------------------------------------------------------------------------------------
def test_case_table_covers_the_edges(orc):
    crossing = []
    for name, (n, nb, is3d, gp, kw) in CASES.items():
        flags, div, sys = build_case(orc, name)
        assert sys.ncomp >= 1, name
        assert sys.pivot_margin > 5e-7, "%s: a pivot is too close to its guard threshold for fp32" % name
        if gp:
            crossing += crossing_small_components(sys, gp)
            assert sys.is3d or gp < nb, name
    assert crossing.count(3) >= 2 and crossing.count(4) >= 2, crossing
    f, d, s = build_case(orc, "3d-nx>ny-gp1")
    assert (s.size == 5).any() and (s.size == 3).any() and (s.size == 4).any() and (s.size == 2).any()
    assert s.guarded.any(), "no chain reaches the pivot guard"
    assert (np.bincount(s.cid) > 1000).any()
    f, d, s = build_case(orc, "3d-ny>nx-gp7-empty")
    assert (f == 4).any()


@pytest.mark.parametrize("name", list(CASES))
def test_sweep_emulation_within_kappa(orc, name):
    """The kernel's fp32 sweep arithmetic, emulated, stays within KAPPA / 8 of the float64 preconditioner; an
    unmasked cross-CTA z- term does not, wherever a small component crosses a chunk boundary."""
    flags, div, sys = build_case(orc, name)
    gp = CASES[name][3]
    r = sys.gather(div)
    z64 = sys.precond(r)
    S = sys.precond(np.abs(r))
    z32 = R.emulate_sweep_fp32(sys, r, groups=gp)
    err = np.abs(z32 - z64)
    assert np.all(err <= KAPPA / 8 * S), (err / np.maximum(S, 1e-300)).max()
    if crossing_small_components(sys, gp):
        bad = R.emulate_sweep_fp32(sys, r, groups=gp, masked=False)
        assert np.any(np.abs(bad - z64) > KAPPA * S)


def _per_component_err(sys, got, want):
    """max|got - want| / max|want| on each component's cells."""
    g, w = sys.gather(got), sys.gather(want)
    err = np.zeros(sys.ncomp)
    np.maximum.at(err, sys.cid, np.abs(g - w))
    scale = np.zeros(sys.ncomp)
    np.maximum.at(scale, sys.cid, np.abs(w))
    return err / np.maximum(scale, 1e-30)


FREEZE_CASE = "3d-nx>ny-gp3"
FREEZE_CAP = 4                                  # maxIter of the freeze test: 5 iterations, bound TAU[4]


def freeze_reference(sys, div):
    """(tol, p64, iterations per component, early): a tol at which the components of fewer than 20 cells that
    the float64 loop solves exactly within FREEZE_CAP iterations stop, every other component runs all
    FREEZE_CAP + 1, no rr up to a stop comes within 2x of tol^2, and at least one component stops BEFORE its exact
    solve ('early').  For each early component the next iterate differs from the one it stopped at by more than
    10 TAU[FREEZE_CAP] of its scale, so a component that kept iterating is detectably wrong."""
    cap = FREEZE_CAP
    _, _, _, hist = sys.solve(div, 1e-30, cap + 1, history=True)
    rr0 = sys.comp_sum(sys.gather(div) ** 2)
    traj = np.stack([rr0] + [rr for _, rr in hist[:cap + 1]])     # [iteration][component]
    stops = (sys.size < 20) & (traj[1:cap + 1] < 1e-8 * rr0).any(axis=0)
    top = traj[:, ~stops].min() / 8
    for tol2 in top * np.logspace(0, -6, 97):
        # above the fp32 rounding floor of a solved component, and a clean stop for every component
        if not (tol2 > 1e-9 * rr0[stops].max() and _clear_stops(traj, tol2, stops, margin=2.0)):
            continue
        tol = float(np.float32(np.sqrt(tol2)))
        want, its, rr = sys.solve(div, tol, cap)
        early = (its < cap + 1) & (rr > 1e-8 * rr0)
        if not early.any():
            continue
        assert np.array_equal(its < cap + 1, stops)
        for c in np.flatnonzero(early):
            on = sys.cid == c
            a, b = sys.gather(hist[its[c] - 1][0])[on], sys.gather(hist[its[c]][0])[on]
            assert np.abs(b - a).max() > 10 * TAU[cap] * np.abs(a).max(), c
        return tol, want, its, early
    raise AssertionError("no tol stops a component before its exact solve while the large ones run on")


@pytest.mark.parametrize("precond", ["none", "ic0"])
def test_oracle_freeze_within_tau(orc, precond):
    """The freeze case through the oracle: the same iteration count, every component within TAU[FREEZE_CAP] / 8
    of its own float64 iterate."""
    flags, div, sys = build_case(orc, FREEZE_CASE, precond)
    tol, want, its, early = freeze_reference(sys, div)
    p = np.zeros(flags.shape, np.float32)
    orc.solveLinearSystemPCG(p, flags, div, True, tol, FREEZE_CAP, precond)
    assert orc.last_pcg_iters == its.max() == FREEZE_CAP + 1
    assert _per_component_err(sys, p, want).max() <= TAU[FREEZE_CAP] / 8


def _clear_stops(traj, tol2, should_stop, margin=4.0):
    """traj: rr per [iteration][component] (row 0: before the first).  True when exactly the components
    `should_stop` fall below tol2, and every rr up to a component's stop is more than `margin` times away."""
    for c in range(traj.shape[1]):
        below = np.flatnonzero(traj[:, c] <= tol2)
        if bool(len(below)) != bool(should_stop[c]):
            return False
        seen = traj[:below[0] + 1 if len(below) else None, c]
        with np.errstate(divide="ignore"):
            if np.any(np.abs(np.log2(seen / tol2)) <= np.log2(margin)):
                return False
    return True


def fixed_count_reference(sys, div, k):
    """(tol, p64 after k + 1 iterations, iterations, components compared).  A component of a few cells is solved
    exactly within its size in iterations; past that its r is rounding noise (NaN in fp32 soon after), so tol is
    put far below every rr of the components still running ('live') and far above the rr of an exactly solved
    one: those stop when they are solved, the live ones run all k + 1 iterations."""
    _, _, _, hist = sys.solve(div, 1e-30, k, history=True)
    rr0 = sys.comp_sum(sys.gather(div) ** 2)
    traj = np.stack([rr0] + [h[1] for h in hist])
    live = traj.min(axis=0) > 1e-8 * rr0
    top = 1e-3 * traj[:, live].min()
    tol2 = next(t for t in top * np.logspace(0, -8, 65) if _clear_stops(traj, t, ~live))
    tol = float(np.float32(np.sqrt(tol2)))
    want, it, _ = sys.solve(div, tol, k)
    assert np.all(it[live] == k + 1)
    return tol, want, it, live


@pytest.mark.parametrize("precond", ["none", "ic0"])
@pytest.mark.parametrize("name", ITER_CASES)
def test_oracle_iterates_within_tau(orc, name, precond):
    flags, div, sys = build_case(orc, name, precond)
    is3d = CASES[name][2]
    for k in TAU:
        tol, want, it, live = fixed_count_reference(sys, div, k)
        p = np.zeros(flags.shape, np.float32)
        orc.solveLinearSystemPCG(p, flags, div, is3d, tol, k, precond)
        assert orc.last_pcg_iters == k + 1 == it.max()
        assert live[np.argmax(sys.size)] and not np.isnan(p).any()
        e = _per_component_err(sys, p, want)
        assert e.max() <= TAU[k] / 8, (k, e.max())


# ---------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    """A context of its own; the planes-per-CTA override is reset at teardown."""
    import torch
    from fluidnet_b200 import tfluids
    from fluidnet_b200._lib import Grid
    dev = torch.cuda.current_device()
    saved = tfluids._contexts.get(dev)
    ctx = tfluids.Context(dev)
    tfluids._contexts[dev] = ctx
    ctx.lib.tfl_debug_pcg_groups.argtypes = [C.c_void_p, C.c_int]
    ctx.lib.tfl_debug_pcg_precond.argtypes = [C.c_void_p, C.POINTER(Grid), C.POINTER(Grid), C.POINTER(Grid),
                                              C.c_int, C.c_int, C.POINTER(C.c_int32)]
    try:
        yield ctx
    finally:
        torch.cuda.synchronize()
        ctx.lib.tfl_debug_pcg_groups(ctx.h, 0)
        if saved is None:
            tfluids._contexts.pop(dev, None)
        else:
            tfluids._contexts[dev] = saved
        ctx.lib.tfl_destroy(ctx.h)
        ctx.h = None


def set_groups(ctx, gp):
    assert ctx.lib.tfl_debug_pcg_groups(ctx.h, gp or 0) == 0


def gpu_precond(ctx, flags, r, is3d, precond="ic0"):
    """(z, (NYP, planes per CTA, chunks, cooperative grid))."""
    import torch
    from fluidnet_b200 import tfluids
    f = torch.from_numpy(flags).cuda()
    d = torch.from_numpy(np.ascontiguousarray(r, np.float32)).cuda()
    z = torch.full_like(f, 7.0)                                    # must be overwritten everywhere
    geo = (C.c_int32 * 4)()
    ctx.use_current_stream()
    ctx.check(ctx.lib.tfl_debug_pcg_precond(ctx.h, C.byref(tfluids._grid(z)), C.byref(tfluids._grid(f)),
                                            C.byref(tfluids._grid(d)), 1 if is3d else 0,
                                            {"none": 0, "ilu0": 1, "ic0": 2}[precond], geo))
    return z.cpu().numpy(), tuple(geo)


def gpu_solve(flags, div, is3d, tol, max_iter, precond):
    from gpu_backend import GpuBackend
    g = GpuBackend()
    p = np.full(flags.shape, 3.0, np.float32)
    g.solveLinearSystemPCG(p, flags, div, is3d, tol, max_iter, precond)
    return p, g.last_pcg_iters


def check_precond(sys, z, r_nat, what):
    r = sys.gather(r_nat)
    z64 = sys.precond(r)
    S = sys.precond(np.abs(r))
    err = np.abs(sys.gather(z) - z64)
    ratio = (err / np.maximum(S, 1e-300)).max() if len(err) else 0.0
    assert np.all(err <= KAPPA * S), "%s: max err/S %g (KAPPA %g)" % (what, ratio, KAPPA)
    outside = np.ones(z.size, bool)
    outside[sys.cells] = False
    assert np.all(z.reshape(-1)[outside].view(np.uint32) == 0), "%s: nonzero outside the systems" % what
    return ratio


@pytest.mark.gpu
@pytest.mark.parametrize("precond", ["ic0", "ilu0"])
@pytest.mark.parametrize("name", list(CASES))
def test_gpu_preconditioner_per_voxel(orc, lib, name, precond):
    flags, div, sys = build_case(orc, name, "ic0")
    n, nb, is3d, gp, kw = CASES[name]
    set_groups(lib, gp)
    z, (nyp, planes, chunks, grid) = gpu_precond(lib, flags, div, is3d, precond)
    ny = n[1]
    assert nyp == (ny + 31) // 32 * 32
    if gp:
        assert planes == min(gp, (1024 - 64) // nyp, nb * n[2])
    if name == "2d-ny960":
        assert (nyp, planes) == (960, 1)
    if name == "3d-column-multichunk":
        assert chunks > grid, (chunks, grid)                        # CTAs own several chunks
    ratio = check_precond(sys, z, div, name)
    print("%s %s: max err/S %.3g, geometry NYP %d GP %d chunks %d grid %d" % (name, precond, ratio, nyp, planes,
                                                                           chunks, grid))


@pytest.mark.gpu
def test_gpu_preconditioner_none_is_identity(orc, lib):
    flags, div, sys = build_case(orc, "3d-nx>ny-gp3")
    set_groups(lib, 3)
    z, _ = gpu_precond(lib, flags, div, True, "none")
    want = sys.scatter(sys.gather(div), np.float32)
    assert np.array_equal(z.view(np.uint32), want.view(np.uint32))


@pytest.mark.gpu
def test_gpu_preconditioner_full_size(orc, lib):
    from fluidnet_b200 import synth
    nn = 128
    flags = synth.make_flags(nn, nn, nn, True, nb=1, geometry=True, exotic=False)
    div = make_div(orc, flags, True, seed=7)
    sys = R.System(orc, flags, True, "ic0")
    assert sys.pivot_margin > 5e-7
    set_groups(lib, 0)
    z, (nyp, planes, chunks, grid) = gpu_precond(lib, flags, div, True)
    assert (nyp, planes) == (128, 7) and chunks == 19
    print("128^3: max err/S %.3g" % check_precond(sys, z, div, "128^3"))


@pytest.mark.gpu
def test_gpu_ny961_refused(orc, lib):
    from fluidnet_b200._lib import TflError
    flags = make_flags(orc, (8, 961, 1), 1, False, small=False)
    set_groups(lib, 0)
    with pytest.raises(TflError, match="ny > 960"):
        gpu_precond(lib, flags, make_div(orc, flags, False), False)


@pytest.mark.gpu
def test_gpu_preconditioner_deterministic(orc, lib):
    """Bit-identical z on repeated calls, and after solves on other shapes (new progress-word epochs, and a
    reallocation of the progress words by the many-chunk column)."""
    flags, div, sys = build_case(orc, "3d-ny>nx-gp3")
    set_groups(lib, 3)
    z0, _ = gpu_precond(lib, flags, div, True)
    z1, _ = gpu_precond(lib, flags, div, True)
    assert np.array_equal(z0.view(np.uint32), z1.view(np.uint32))
    for other in ("2d-nb5-gp2", "3d-column-multichunk", "3d-cube-gp2"):
        f2, d2, _ = build_case(orc, other)
        set_groups(lib, CASES[other][3])
        gpu_solve(f2, d2, CASES[other][2], 1e-30, 2, "ic0")
        set_groups(lib, 3)
        z2, _ = gpu_precond(lib, flags, div, True)
        assert np.array_equal(z0.view(np.uint32), z2.view(np.uint32)), other


@pytest.mark.gpu
@pytest.mark.parametrize("precond", ["none", "ilu0", "ic0"])
@pytest.mark.parametrize("name", ITER_CASES)
def test_gpu_fixed_count_iterates(orc, lib, name, precond):
    flags, div, sys = build_case(orc, name, "none" if precond == "none" else "ic0")
    n, nb, is3d, gp, kw = CASES[name]
    set_groups(lib, gp)
    worst = 0.0
    for k in TAU:
        tol, want, its, live = fixed_count_reference(sys, div, k)
        p, it = gpu_solve(flags, div, is3d, tol, k, precond)
        assert it == k + 1 == its.max()
        e = _per_component_err(sys, p, want)
        assert e.max() <= TAU[k], "%s %s maxIter %d: %g > %g" % (name, precond, k, e.max(), TAU[k])
        assert np.all(p[sys.scatter(np.ones(sys.m)) == 0] == 0)
        worst = max(worst, e.max() / TAU[k])
    print("%s %s: max err/(tau max|p|) %.3g" % (name, precond, worst))


@pytest.mark.gpu
@pytest.mark.parametrize("precond", ["none", "ic0"])
def test_gpu_components_freeze_independently(orc, lib, precond):
    flags, div, sys = build_case(orc, FREEZE_CASE, "none" if precond == "none" else "ic0")
    tol, want, its, early = freeze_reference(sys, div)
    set_groups(lib, CASES[FREEZE_CASE][3])
    p, it = gpu_solve(flags, div, True, tol, FREEZE_CAP, precond)
    assert it == its.max() == FREEZE_CAP + 1
    e = _per_component_err(sys, p, want)
    assert e.max() <= TAU[FREEZE_CAP], e.max()
    print("freeze %s: %d components stop early, max err/(tau max|p|) %.3g" % (
        precond, early.sum(), e.max() / TAU[FREEZE_CAP]))
