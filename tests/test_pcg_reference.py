"""The float64 PCG restatement (tests/pcg_reference.py) pinned on its own definition, on small grids: the
wavefront-vectorised factor and solves equal the cell-by-cell loops, the factor is IC(0) (R^T R = A on A's
sparsity pattern), z = M^-1 r solves M z = r, and the loop run to convergence solves setupLaplacian's system."""
import numpy as np
import pytest
import scipy.sparse as sp

import pcg_cases
import pcg_reference as R


def _systems(orc):
    for is3d in (True, False):
        for empty in (False, True):
            flags, U, div = pcg_cases.make(orc, is3d, nb=2, n=(12, 11, 10), empty=empty)
            yield flags, div, R.System(orc, flags, is3d, "ic0"), is3d


def _matrices(sys):
    """(A, L) as scipy matrices over the compact cells; M = L L^T with L = R^T (L_ii = 1 / pre_i,
    L_ik = -pre_k for a lower neighbour k).  Rows of un-preconditioned cells of L are the identity."""
    m = sys.m
    rows, cols, vals = [], [], []
    lrows, lcols, lvals = [], [], []
    for t in range(sys.lo.shape[0]):
        for nb in (sys.lo[t], sys.hi[t]):
            ok = np.flatnonzero(nb < m)
            rows += list(ok); cols += list(nb[ok]); vals += [-1.0] * len(ok)
        ok = np.flatnonzero((sys.lo[t] < m) & sys.use_pre)
        lrows += list(ok); lcols += list(sys.lo[t][ok]); lvals += list(-sys.pre[sys.lo[t][ok]])
    A = sp.csr_matrix((vals, (rows, cols)), shape=(m, m)) + sp.diags(sys.diag)
    d = np.where(sys.use_pre, 1.0 / np.where(sys.use_pre, sys.pre[:m], 1.0), 1.0)
    L = sp.csr_matrix((lvals, (lrows, lcols)), shape=(m, m)) + sp.diags(d)
    return A, L


def test_vectorised_equals_cell_loop(orc):
    for flags, div, sys, is3d in _systems(orc):
        pre = sys.factor_cells()
        assert np.abs(pre - sys.pre).max() <= 1e-13 * np.abs(pre).max()
        r = sys.gather(div)
        for v in (r, np.abs(r)):
            want = sys.precond_cells(v, pre)
            got = sys.precond(v)
            assert np.abs(got - want).max() <= 1e-13 * np.abs(want).max()
        assert sys.use_pre.any() and not sys.use_pre.all()


def test_factor_is_ic0_of_A(orc):
    """R^T R = A on A's sparsity pattern at every row whose pivot is not guarded; M z = r."""
    for flags, div, sys, is3d in _systems(orc):
        A, L = _matrices(sys)
        M = (L @ L.T).tocsr()
        rows = np.flatnonzero(sys.use_pre & ~sys.guarded)
        pattern = A[rows].tocoo()
        diff = np.asarray(M[rows][pattern.row, pattern.col]).ravel() - pattern.data
        assert np.abs(diff).max() < 1e-12
        r = sys.gather(div)
        z = sys.precond(r)
        on = sys.use_pre
        assert np.abs((M @ np.where(on, z, 0.0))[on] - r[on]).max() <= 1e-12 * np.abs(r).max()
        assert np.array_equal(z[~on], r[~on])


def test_pivot_guard_on_a_chain(orc):
    """A 1-cell-wide chain of 6 along x: every pivot is 1 exactly but the last, 0, which the guard replaces by
    its diagonal; the margin to the guard threshold is 1e-6 d."""
    flags = np.ones((1, 1, 8, 8, 12), np.float32)
    orc.emptyDomain(flags, True, 1)
    flags[0, 0, 1:7, 1:7, 1:11] = 2
    flags[0, 0, 4, 4, 3:9] = 1
    sys = R.System(orc, flags, True, "ic0")
    assert sys.m == 6 and sys.guarded.sum() == 1 and sys.guarded[-1]
    assert np.array_equal(sys.pivot, [1, 1, 1, 1, 1, 0])
    assert sys.pivot_margin == pytest.approx(1e-6)


def test_converged_loop_solves_the_system(orc):
    """Run to convergence, p (mean removed) solves A p = div - mean(div) per component; the iteration counts are
    the reference's semantics (maxIter + 1 iterations at most)."""
    for flags, div, sys, is3d in _systems(orc):
        p, it, rr = sys.solve(div, 1e-6, 1000)
        assert np.all(rr <= np.float32(1e-6) ** 2) and it.max() <= 1001
        A, _ = _matrices(sys)
        r = sys.gather(div)
        rhs = r - (sys.comp_sum(r) / sys.size)[sys.cid]
        x = sys.gather(p)
        assert np.abs(sys.comp_sum(x)).max() < 1e-9
        # pure Neumann components (A 1 = 0); one that touches Empty cells is shifted by the mean removal
        neumann = (sys.comp_sum(np.abs(A @ np.ones(sys.m))) == 0)[sys.cid]
        assert neumann.any()
        assert np.abs(A @ x - rhs)[neumann].max() < 1e-5 * np.abs(r).max()
        assert np.abs(A @ x - sys.apply_A(x)).max() < 1e-12 * np.abs(x).max()
        _, it3, _ = sys.solve(div, 1e-30, 3)
        assert it3.max() == 4
