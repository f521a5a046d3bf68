"""The Jacobi solve run to a tolerance on the device (tfl_solve_linear_system_jacobi_dev, and the direct call with
pTol > 0): p bit for bit and the iteration count of the oracle's host loop, the residual within 1e-6, on the resident
path (k_jacobi_resident<4, true>, one cooperative launch) and on the chunked path (gated sweeps, k_jacobi_residual,
host-read chunks of 8, 16, 32, ... sweeps or a conditional WHILE node in a capture).  Also: the residual's fixed
summation order, no host wait, replays of a captured solve, and the launch tally against the profiler."""
import time

import numpy as np
import pytest
import torch

import oracle
from cases import bits_equal, describe_diff
from fluidnet_b200 import synth
from step_cases import ctx, run_in_child, tally_and_kernels

# (nz, ny, nx) -> the path the tolerance solve takes there
GRIDS = {
    "16x32x128": ((16, 32, 128), "resident"),
    "4x8x128": ((4, 8, 128), "resident"),            # the smallest resident grid: one block, nz = 4
    "6x10x13": ((6, 10, 13), "chunked"),             # nx % 4 != 0: k_jacobi_iter
    "2d-40x36": ((1, 40, 36), "chunked"),            # 2-D: k_jacobi_iter4<false>
    "32x128x1024": ((32, 128, 1024), "chunked"),     # above 3 x 2^20 cells: k_jacobi_march
}
# The host-read chunks end after 8, 24, 56 sweeps; the captured loop body is 16 sweeps.
STOP_SWEEPS = (1, 2, 7, 8, 9, 15, 16, 17, 23, 24, 25, 55, 56, 57)


def scene(shape, nb=1, seed=5):
    """(flags, div, is3d): obstacles, empty and outflow cells, the divergence of a smooth velocity with wall BCs;
    batch entry b's divergence scaled by 4^-b, so the entries converge after different sweeps."""
    nz, ny, nx = shape
    is3d = nz > 1
    flags = synth.make_flags(nx, ny, nz, is3d, nb=nb, geometry=True, exotic=nz != 4)
    U = synth.make_smooth_velocity(flags, is3d, amp=1.0, seed=seed)
    orc = oracle.Oracle()
    orc.setWallBcsForward(U, flags)
    div = orc.velocityDivergenceForward(U, flags)
    scale = (np.float32(0.25) ** np.arange(nb, dtype=np.float32)).reshape(nb, 1, 1, 1, 1)
    return flags, np.ascontiguousarray((div * scale).astype(np.float32)), is3d


def gpu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def solve(flags, div, is3d, tol, max_iter, dev):
    """(p, residual as float32, iterations) of the direct call or of the _dev call, p starting at 9."""
    from fluidnet_b200 import tfluids
    p = torch.full(div.shape, 9.0, device="cuda")
    f, d = gpu(flags), gpu(div)
    if dev:
        r, it = tfluids.solveLinearSystemJacobiDevice(p, f, d, is3d, tol, max_iter)
        return p.cpu().numpy(), np.float32(r.item()), int(it.item())
    r = tfluids.solveLinearSystemJacobi(p, f, d, is3d, tol, max_iter)
    return p.cpu().numpy(), np.float32(r), tfluids.solveLinearSystemJacobi.last_iterations


def oracle_solve(orc, flags, div, is3d, tol, max_iter):
    p = np.full(div.shape, 9.0, np.float32)
    r = orc.solveLinearSystemJacobi(p, flags, div, is3d, tol, max_iter)
    return p, np.float32(r), orc.last_jacobi_iters


def check(got, want, what):
    assert bits_equal(got[0], want[0]), "%s: p %s" % (what, describe_diff(got[0], want[0]))
    assert got[2] == want[2], (what, "iterations", got[2], want[2])
    assert abs(float(got[1]) - float(want[1])) <= 1e-6 * abs(float(want[1])), (what, "residual", got[1], want[1])


def residual_sequence(flags, div, is3d, sweeps):
    """The residual after 1 .. sweeps sweeps (fixed-count solves)."""
    from fluidnet_b200 import tfluids
    f, d = gpu(flags), gpu(div)
    p = torch.empty_like(d)
    return [tfluids.solveLinearSystemJacobi(p, f, d, is3d, 0.0, k) for k in range(1, sweeps + 1)]


def tol_stopping_after(seq, m):
    """A pTol whose solve stops after sweep m (iterations m - 1), half way (geometrically) between the residual there
    and the smallest one before it, or None when no such pTol keeps clear of a tie."""
    lo = seq[m - 1]
    hi = min(seq[:m - 1]) if m > 1 else 4.0 * lo
    if not (lo > 0 and hi > lo * (1 + 1e-3)):
        return None
    return float(np.float32(np.sqrt(lo * hi)))


@pytest.mark.gpu
@pytest.mark.parametrize("grid", list(GRIDS))
def test_matches_the_oracle(orc, grid):
    shape, _ = GRIDS[grid]
    flags, div, is3d = scene(shape)
    seq = residual_sequence(flags, div, is3d, max(STOP_SWEEPS))
    tols = {m: tol_stopping_after(seq, m) for m in STOP_SWEEPS}
    assert sum(t is None for t in tols.values()) <= 2, tols
    cases = [(t, 1000, "stops after sweep %d" % m) for m, t in tols.items() if t is not None]
    cases += [(1e-30, n, "never meets pTol, maxIter %d" % n) for n in (1, 2, 30, 31)]
    for tol, max_iter, what in cases:
        want = oracle_solve(orc, flags, div, is3d, tol, max_iter)
        if what.startswith("stops"):
            assert want[2] == int(what.split()[-1]) - 1, (what, want[2])
        for dev in (False, True):
            how = "%s %s (%s)" % (grid, what, "_dev" if dev else "direct")
            check(solve(flags, div, is3d, tol, max_iter, dev), want, how)


@pytest.mark.gpu
@pytest.mark.parametrize("grid", ["16x32x128", "6x10x13"])
@pytest.mark.parametrize("nb", [1, 2, 3])
def test_batches_stop_on_the_largest_norm(orc, grid, nb):
    shape, _ = GRIDS[grid]
    flags, div, is3d = scene(shape, nb)
    seq = residual_sequence(flags, div, is3d, 25)
    for m in (9, 25):
        tol = tol_stopping_after(seq, m)
        assert tol is not None, (m, seq)
        want = oracle_solve(orc, flags, div, is3d, tol, 1000)
        assert want[2] == m - 1
        for b in range(1, nb):          # entry b alone would have stopped earlier: entry 0 decides
            assert oracle_solve(orc, flags[b:b + 1], div[b:b + 1], is3d, tol, 1000)[2] < want[2]
        for dev in (False, True):
            check(solve(flags, div, is3d, tol, 1000, dev), want, "%s nb %d stop %d" % (grid, nb, m))


@pytest.mark.gpu
@pytest.mark.parametrize("grid", ["128x128x128", "32x128x1024"])
def test_identical_solves_give_identical_residual_bits(grid):
    shape = tuple(int(v) for v in grid.split("x"))
    flags, div, is3d = scene(shape)
    runs = [solve(flags, div, is3d, 1e-30, 60, dev=True) for _ in range(2)]
    assert runs[0][1].tobytes() == runs[1][1].tobytes(), runs
    assert bits_equal(runs[0][0], runs[1][0]) and runs[0][2] == runs[1][2] == 60


def busy_stream_returns(call):
    """(seconds `call` took, whether the stream was still busy when it returned) with ~50 ms of matmuls ahead."""
    stream = torch.cuda.current_stream()
    a = torch.randn(4096, 4096, device="cuda")
    b = torch.randn(4096, 4096, device="cuda") / 64.0
    a = a @ b
    stream.synchronize()
    for _ in range(20):
        a = a @ b
    t0 = time.perf_counter()
    call()
    took = time.perf_counter() - t0
    busy = not stream.query()
    stream.synchronize()
    return took, busy


@pytest.mark.gpu
def test_device_call_and_direct_call_without_outputs_do_not_wait():
    from fluidnet_b200 import tfluids
    from fluidnet_b200.tfluids import _grid
    flags, div, is3d = scene((128, 128, 128))          # resident
    f, d = gpu(flags), gpu(div)
    p = torch.zeros_like(d)
    c = ctx()
    out = {}
    direct = lambda: c.check(c.lib.tfl_solve_linear_system_jacobi(c.h, _grid(p), _grid(f), _grid(d), 1, 1e-5, 100000,
                                                                 None, None))
    device = lambda: out.update(r=tfluids.solveLinearSystemJacobiDevice(p, f, d, is3d, 1e-5, 100000))
    device()
    direct()
    for name, call in (("_dev", device), ("direct, no outputs", direct)):
        took, busy = busy_stream_returns(call)
        assert busy, "%s: the queued work finished before the call returned: nothing was measured" % name
        assert took < 0.02, (name, took)
    res, it = out["r"]
    got = tfluids.solveLinearSystemJacobi(p, f, d, is3d, 1e-5, 100000)
    assert np.float32(got).tobytes() == res.cpu().numpy().tobytes()
    assert tfluids.solveLinearSystemJacobi.last_iterations == int(it.item()) > 100


@pytest.mark.gpu
@pytest.mark.parametrize("grid", ["16x32x128", "6x10x13"])
def test_captured_solve_replays_like_direct_calls(grid):
    from fluidnet_b200 import tfluids
    from fluidnet_b200.tfluids import TflError
    shape, _ = GRIDS[grid]
    flags, div0, is3d = scene(shape)
    # closed fluid pockets keep the residual above 1e-4 at full scale; these scales converge, after different sweeps
    tol, max_iter = 1e-4, 20000
    f, d = gpu(flags), gpu(div0)
    p = torch.zeros_like(d)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        tfluids.solveLinearSystemJacobiDevice(p, f, d, is3d, tol, max_iter)     # sizes the scratch arena
        side.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=side):
            with pytest.raises(TflError, match="tfl_solve_linear_system_jacobi_dev"):
                tfluids.solveLinearSystemJacobi(p, f, d, is3d, tol, max_iter)
            res, it = tfluids.solveLinearSystemJacobiDevice(p, f, d, is3d, tol, max_iter)
    torch.cuda.synchronize()
    seen = []
    for scale in (0.05, 0.02, 0.01):
        d.copy_(gpu(div0 * np.float32(scale)))
        graph.replay()
        torch.cuda.synchronize()
        got = (p.cpu().numpy(), np.float32(res.item()), int(it.item()))
        want = solve(flags, div0 * np.float32(scale), is3d, tol, max_iter, dev=False)
        assert bits_equal(got[0], want[0]), (grid, scale, describe_diff(got[0], want[0]))
        assert got[1].tobytes() == want[1].tobytes() and got[2] == want[2], (grid, scale, got[1:], want[1:])
        seen.append(got[2])
    assert len(set(seen)) == 3 and max(seen) < max_iter, seen


@pytest.mark.gpu
def test_refusals():
    from fluidnet_b200 import tfluids
    from fluidnet_b200.tfluids import TflError
    flags, div, is3d = scene((6, 10, 13))
    f, d = gpu(flags), gpu(div)
    p = torch.zeros_like(d)
    c = ctx()
    l0 = c.launch_count()
    with pytest.raises(TflError, match="maxIter < 1"):
        tfluids.solveLinearSystemJacobiDevice(p, f, d, is3d, 1e-5, 0)
    assert c.launch_count() == l0


def profile_solve(shape, tol, max_iter):
    """(tally, {kernel: count}) of one _dev solve, in a child interpreter (run_in_child)."""
    from fluidnet_b200 import tfluids
    flags, div, is3d = scene(tuple(shape))
    f, d = gpu(flags), gpu(div)
    p = torch.zeros_like(d)
    tally, seen = tally_and_kernels(ctx(), lambda: tfluids.solveLinearSystemJacobiDevice(p, f, d, is3d, tol, max_iter))
    return tally, dict(seen)


@pytest.mark.gpu
@pytest.mark.parametrize("grid", list(GRIDS))
@pytest.mark.parametrize("max_iter", [3, 40])
def test_path_and_launch_tally(grid, max_iter):
    shape, path = GRIDS[grid]
    tally, seen = run_in_child("test_gpu_jacobi_tolerance", "t.profile_solve(%r, 1e-30, %d)" % (list(shape), max_iter))
    assert tally == sum(seen.values()), (tally, seen)
    names = " ".join(seen)
    count = lambda s: sum(n for k, n in seen.items() if s in k)
    assert count("k_jacobi_mask") == 1, seen
    if path == "resident":
        assert count("k_jacobi_resident<4, true>") == 1 and tally == 2, seen
    else:
        assert "k_jacobi_resident" not in names, seen
        assert count("k_jacobi_residual") == max_iter and count("k_jacobi_copy_back") == 1, seen
        assert tally == 2 + 2 * max_iter, (tally, seen)
