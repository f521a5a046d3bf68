"""Float64 restatement of the PCG solve (tfl_pcg.cu, oracle/tfluids_oracle.c: orc_pcg), per connected component
and in the system's lexicographic (k, j, i) order.

* The matrix is setupLaplacian's (generic/tfluids.cu:909-1095): the diagonal counts the non-obstacle neighbours,
  fluid neighbours get -1.  Components come from the oracle's flood fill (pinned on the reference); size 1 is
  skipped, below 5 cells no preconditioner is used.
* IC(0) of the 7-point matrix: R_ii = sqrt(d_i - sum over the lower neighbours k of R_ki^2), R_ki = -1 / R_kk, with
  the pivot guard `e > 1e-6 d else d` of the oracle and the kernel.  M = R^T R; ilu0 and ic0 are the same operator.
* The loop is the reference's: `while (rr > tol^2 && iter <= maxIter)`, x0 = 0, beta = 0 on the first iteration,
  clampToEpsilon on both divisions, the mean of x removed per component.

`System` holds every batch entry and component at once on the in-system cells (compact arrays; index m is a
zero sentinel for a missing neighbour).  The triangular solves exist twice: `*_cells` loops over the cells of each
component one by one (small grids), the default processes wavefronts i + j + k = s together (dependencies are
only on -x, -y, -z), so that 128^3 takes seconds.  `emulate_sweep_fp32` repeats the kernel's fp32 sweep
arithmetic (operand order and FMA contractions of k_sweep's SASS) on the same wavefronts, to calibrate bounds."""
import numpy as np

GUARD = 1e-6
EPS = 1.17549435e-38                                     # clampToEpsilon, generic/tfluids.cu:1153-1163


def clamp_eps(v):
    v = np.asarray(v, np.float64)
    return np.where(np.abs(v) < EPS, np.where(v < 0, -EPS, EPS), v)


class System:
    """The setupLaplacian systems of a [nb][1][nz][ny][nx] flag grid (precond: 'none' | 'ilu0' | 'ic0')."""

    def __init__(self, orc, flags, is3d, precond="ic0"):
        nb, _, nz, ny, nx = flags.shape
        self.shape, self.is3d = flags.shape, is3d
        f = flags[:, 0].astype(np.int64)
        n = nz * ny * nx
        comp = np.full(nb * n, -1, np.int64)
        sizes = []
        for b in range(nb):
            c, s = orc.findConnectedFluidComponents(flags, is3d, b)
            c = c.reshape(-1).astype(np.int64)
            comp[b * n:(b + 1) * n] = np.where(c >= 0, c + len(sizes), -1)
            sizes.extend(int(v) for v in s)
        sizes = np.array(sizes, np.int64)
        insys = comp >= 0
        insys[insys] = sizes[comp[insys]] >= 2
        cells = np.flatnonzero(insys)                    # natural flat index of each system cell, lexicographic
        m = len(cells)
        self.cells, self.m = cells, m
        # dense component ids of the systems (components of >= 2 cells), in the reference's order
        sys_comps, self.cid = np.unique(comp[cells], return_inverse=True)
        self.ncomp = len(sys_comps)
        self.size = sizes[sys_comps]
        self.comp_of_component = sys_comps
        self.use_pre = (precond != "none") & (self.size[self.cid] >= 5)
        self.batch = cells // n
        rem = cells % n
        self.k, self.j, self.i = rem // (ny * nx), (rem // nx) % ny, rem % nx
        ff = f.reshape(-1)
        compact = np.full(nb * n + 1, m, np.int64)
        compact[cells] = np.arange(m)
        steps = [1, nx] + ([nx * ny] if is3d else [])
        diag = np.zeros(m, np.float64)
        lo, hi = [], []
        for st in steps:
            for sign, out in ((-1, lo), (1, hi)):
                nbf = ff[cells + sign * st]
                diag += (nbf & 2) == 0
                out.append(np.where((nbf & 1) != 0, compact[cells + sign * st], m))
        self.diag = diag
        self.lo = np.stack(lo)                            # [-x, -y, (-z)] compact index or m
        self.hi = np.stack(hi)                            # [+x, +y, (+z)]
        s = self.i + self.j + self.k
        order = np.argsort(s, kind="stable")
        bounds = np.flatnonzero(np.diff(s[order])) + 1
        self.fronts = np.split(order, bounds) if m else []
        self._factor()

    # ---- IC(0) ------------------------------------------------------------------------------------------
    def _factor(self):
        pre = np.zeros(self.m + 1)
        e_all = np.zeros(self.m)
        for q in self.fronts:
            e = self.diag[q] - (pre[self.lo[:, q]] ** 2).sum(axis=0)
            e_all[q] = e
            pre[q] = np.where(self.use_pre[q], 1.0 / np.sqrt(np.where(e > GUARD * self.diag[q], e, self.diag[q])), 0.0)
        self.pre = pre                                    # 1 / R_ii on preconditioned cells, 0 elsewhere
        self.pivot = e_all
        # distance of every pivot from its guard threshold, relative to the diagonal
        p = self.use_pre
        self.pivot_margin = float(np.min(np.abs(e_all[p] - GUARD * self.diag[p]) / self.diag[p])) if p.any() else np.inf
        self.guarded = p & ~(e_all > GUARD * self.diag)

    def factor_cells(self):
        """1 / R_ii, cell by cell and component by component (the plain restatement of _factor)."""
        pre = np.zeros(self.m + 1)
        for c in range(self.ncomp):
            for q in np.flatnonzero(self.cid == c):
                if not self.use_pre[q]:
                    continue
                e = self.diag[q]
                for t in range(self.lo.shape[0]):
                    if self.lo[t, q] < self.m:
                        e -= pre[self.lo[t, q]] ** 2
                pre[q] = 1.0 / np.sqrt(e if e > GUARD * self.diag[q] else self.diag[q])
        return pre

    # ---- z = M^-1 r ----------------------------------------------------------------------------------------
    def precond(self, r):
        """r: compact float64 [m].  Cells of un-preconditioned systems get z = r."""
        pre, up = self.pre, self.use_pre
        y = np.zeros(self.m + 1)
        for q in self.fronts:                             # R^T y = r
            y[q] = (r[q] + (pre[self.lo[:, q]] * y[self.lo[:, q]]).sum(axis=0)) * pre[q]
        z = np.zeros(self.m + 1)
        for q in reversed(self.fronts):                   # R z = y
            z[q] = (y[q] + pre[q] * z[self.hi[:, q]].sum(axis=0)) * pre[q]
        return np.where(up, z[:-1], r)

    def precond_cells(self, r, pre=None):
        pre = self.factor_cells() if pre is None else pre
        z = np.array(r, np.float64)
        for c in range(self.ncomp):
            qs = np.flatnonzero(self.cid == c)
            if not self.use_pre[qs[0]]:
                continue
            y = {}
            for q in qs:
                acc = r[q]
                for t in range(self.lo.shape[0]):
                    if self.lo[t, q] < self.m:
                        acc += pre[self.lo[t, q]] * y[self.lo[t, q]]
                y[q] = acc * pre[q]
            zz = {}
            for q in qs[::-1]:
                acc = 0.0
                for t in range(self.hi.shape[0]):
                    if self.hi[t, q] < self.m:
                        acc += zz[self.hi[t, q]]
                zz[q] = (y[q] + pre[q] * acc) * pre[q]
                z[q] = zz[q]
        return z

    def apply_A(self, v):
        ve = np.append(v, 0.0)
        return self.diag * v - ve[self.lo].sum(axis=0) - ve[self.hi].sum(axis=0)

    # ---- natural layout <-> compact -------------------------------------------------------------------------
    def gather(self, a):
        return np.asarray(a, np.float64).reshape(-1)[self.cells]

    def scatter(self, v, dtype=np.float64):
        out = np.zeros(int(np.prod(self.shape)), dtype)
        out[self.cells] = v
        return out.reshape(self.shape)

    def comp_sum(self, v):
        return np.bincount(self.cid, weights=v, minlength=self.ncomp)

    # ---- the loop -------------------------------------------------------------------------------------------
    def solve(self, div, tol, max_iter, history=False):
        """PCG as the reference runs it, every component on its own.  Returns (p natural float64, iterations per
        component, final rr per component[, [(p, rr per component) after each iteration]])."""
        tol2 = float(np.float32(tol)) ** 2
        r = self.gather(div)
        x = np.zeros(self.m)
        p = np.zeros(self.m)
        rr = self.comp_sum(r * r)
        rz = np.zeros(self.ncomp)
        iters = np.zeros(self.ncomp, np.int64)
        active = (rr > tol2) & (iters <= max_iter)
        hist = []
        with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
            while active.any():
                x, r, p, rz, rr, iters, active = self._iteration(x, r, p, rz, rr, iters, active, tol2, max_iter)
                if history:
                    hist.append((self.scatter(self._mean_removed(x)), rr.copy()))
        out = (self.scatter(self._mean_removed(x)), iters, rr)
        return out + (hist,) if history else out

    def _iteration(self, x, r, p, rz, rr, iters, active, tol2, max_iter):
        """One iteration of every active component (the others keep their state)."""
        a = active[self.cid]
        z = self.precond(r)
        rz_old = rz
        rz = np.where(active, self.comp_sum(r * z), rz)
        iters = iters + active
        beta = np.where(iters > 1, rz / clamp_eps(rz_old), 0.0)
        p = np.where(a, z + beta[self.cid] * p, p)
        w = self.apply_A(p)
        alpha = rz / clamp_eps(self.comp_sum(np.where(a, p * w, 0.0)))
        x = np.where(a, x + alpha[self.cid] * p, x)
        r = np.where(a, r - alpha[self.cid] * w, r)
        rr = np.where(active, self.comp_sum(r * r), rr)
        active = active & (rr > tol2) & (iters <= max_iter)
        return x, r, p, rz, rr, iters, active

    def _mean_removed(self, x):
        return x - (self.comp_sum(x) / self.size)[self.cid]


# ---- fp32 emulation of k_sweep ----------------------------------------------------------------------------------
def _f(v):
    return np.float32(v) if np.isscalar(v) else np.asarray(v, np.float32)


def _fma(a, b, c):
    """fp32 fused multiply-add (the product of two floats is exact in float64; the double rounding of the sum is
    at most one fp32 ulp away in rare ties, far below the bounds this calibrates)."""
    return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(np.float32)


def emulate_sweep_fp32(sys, r, groups=None, masked=True):
    """The factor and one solve sweep of k_sweep in fp32, in its operand order (read from the SASS of
    k_sweep<true> / k_sweep<false>, which tfl_pcg.cu compiles with FMA contraction):
      factor    e = fma(-zm, zm, fma(-ym, ym, fma(-xm, xm, d))); pv = 1 / sqrtf(e or d)  (both correctly rounded)
      forward   y = (((r + xm) + ym) + zm) * pre; passed on as y * (on * pre)
      backward  z = fma(on * pre, (xp + yp) + zp, y) * pre; passed on as z
    The passed values are 0 from cells outside the system and from un-preconditioned cells (on = 0).  In 3-D,
    planes pl = b nz + k with pl % groups == 0 (pl > 0) take their z- term from global memory (the chunk
    boundaries of the pipeline); `masked=False` reproduces the unmasked pre * y read there.
    r: compact [m] array; returns the compact fp32 z."""
    m = sys.m
    nz = sys.shape[2]
    pl = sys.batch * nz + sys.k
    cross = np.zeros(m, bool) if (groups is None or not sys.is3d) else ((pl % groups == 0) & (pl > 0))
    on = _f(sys.use_pre)
    d = _f(sys.diag)
    nlo = sys.lo.shape[0]
    # factor: out = on * pv
    pv = np.zeros(m + 1, np.float32)
    passf = np.zeros(m + 1, np.float32)
    raw_pre = np.zeros(m + 1, np.float32)          # what global memory holds: pv (1 for un-preconditioned cells)
    for q in sys.fronts:
        e = d[q]
        for t in range(nlo):
            v = passf[sys.lo[t, q]]
            if t == 2:
                v = np.where(cross[q], np.where(on[q] != 0, raw_pre[sys.lo[t, q]], _f(0)) if masked
                             else raw_pre[sys.lo[t, q]], v)
            e = _fma(-v, v, e)
        e = np.where(e > _f(1e-6) * d[q], e, d[q])
        p = np.where(on[q] != 0, _f(1) / np.sqrt(e), _f(1))
        raw_pre[q] = p
        passf[q] = on[q] * p
    pre = raw_pre
    rr = _f(np.append(r, 0))
    y = np.zeros(m + 1, np.float32)
    passy = np.zeros(m + 1, np.float32)
    for q in sys.fronts:
        acc = rr[q]
        for t in range(nlo):
            v = passy[sys.lo[t, q]]
            if t == 2:
                g = pre[sys.lo[t, q]] * y[sys.lo[t, q]]
                v = np.where(cross[q], np.where(on[q] != 0, g, _f(0)) if masked else g, v)
            acc = acc + v
        y[q] = acc * pre[q]
        passy[q] = y[q] * (on[q] * pre[q])
    z = np.zeros(m + 1, np.float32)
    for q in reversed(sys.fronts):
        s = z[sys.hi[0, q]] + z[sys.hi[1, q]]
        if sys.hi.shape[0] > 2:
            s = s + z[sys.hi[2, q]]
        z[q] = _fma(on[q] * pre[q], s, y[q]) * pre[q]
    return z[:m]
