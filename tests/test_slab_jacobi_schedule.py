"""The Jacobi sweep schedule of the z-slab step (tfl_slab_jacobi_schedule), checked without a GPU: a float32 numpy
restatement of the sweep runs slab by slab with the exported schedule -- exchanges, shrinking plane ranges, the
divergence and mask valid only on the planes the schedule names -- and must equal the undivided sweep bit for bit on
every owned plane and on the plane below them that the velocity update reads."""
import numpy as np
import pytest

from fluidnet_b200.slab import SlabDecomposition, jacobi_schedule


def _sweep(prev, cur, div, solid, nbr, lo, hi):
    """One sweep on planes [lo, hi) of prev into cur: (p1 + ... + p6 + div) / 6 with the obstacle selects."""
    P = np.pad(prev, 1)
    ctr = P[lo + 1:hi + 1, 1:-1, 1:-1]
    nb = [P[lo + 1:hi + 1, 1:-1, :-2], P[lo + 1:hi + 1, 1:-1, 2:], P[lo + 1:hi + 1, :-2, 1:-1],
          P[lo + 1:hi + 1, 2:, 1:-1], P[lo:hi, 1:-1, 1:-1], P[lo + 2:hi + 2, 1:-1, 1:-1]]
    ps = [np.where(nbr[a][lo:hi], ctr, nb[a]) for a in range(6)]
    with np.errstate(invalid="ignore"):
        r = (ps[0] + ps[1] + ps[2] + ps[3] + ps[4] + ps[5] + div[lo:hi]) / np.float32(6)
    cur[lo:hi] = np.where(solid[lo:hi], np.float32(0), r)


def _problem(gnz, ny, nx, seed):
    rng = np.random.default_rng(seed)
    obst = rng.random((gnz, ny, nx)) < 0.15
    z, y, x = np.meshgrid(np.arange(gnz), np.arange(ny), np.arange(nx), indexing="ij")
    border = (z < 1) | (z > gnz - 2) | (y < 1) | (y > ny - 2) | (x < 1) | (x > nx - 2)
    solid = border | obst
    O = np.pad(obst, 1)
    nbr = [O[1:-1, 1:-1, :-2], O[1:-1, 1:-1, 2:], O[1:-1, :-2, 1:-1], O[1:-1, 2:, 1:-1], O[:-2, 1:-1, 1:-1],
           O[2:, 1:-1, 1:-1]]
    div = rng.standard_normal((gnz, ny, nx)).astype(np.float32)
    return solid, nbr, div


def _undivided(solid, nbr, div, iters):
    a, b = np.zeros_like(div), np.zeros_like(div)
    for _ in range(iters):
        _sweep(a, b, div, solid, nbr, 0, div.shape[0])
        a, b = b, a
    return a


def _slabbed(solid, nbr, div, world, margin, iters):
    gnz = div.shape[0]
    halo = 2 * margin + 2
    decs = [SlabDecomposition(gnz, r, world, halo) for r in range(world)]
    scheds = [jacobi_schedule(gnz, world, r, margin, iters) for r in range(world)]
    nblk = len(scheds[0][1])
    assert all(len(s[1]) == nblk for s in scheds)
    ranks = []
    for d, ((plo, phi, uw), blocks) in zip(decs, scheds):
        loc = lambda a: a[d.zoff:d.zoff + d.nz]
        # divergence and mask are valid on [plo, phi) only: poison the rest
        ldiv = np.full((d.nz,) + div.shape[1:], np.nan, np.float32)
        ldiv[plo:phi] = loc(div)[plo:phi]
        lsolid = np.zeros((d.nz,) + div.shape[1:], bool)
        lsolid[plo:phi] = loc(solid)[plo:phi]
        lnbr = [np.ones_like(lsolid) for _ in range(6)]
        for a in range(6):
            lnbr[a][plo:phi] = loc(nbr[a])[plo:phi]
        # what the divergence reads (U on plo .. phi) and the mask reads (flags plo - 1 .. phi) stay in storage and,
        # across a cut, inside the U exchange
        if d.rank > 0:
            assert plo >= 1 and plo >= d.own_lo - uw
        if d.rank < world - 1:
            assert phi <= d.nz - 1 and phi <= d.own_hi + uw - 1 and phi - 1 < d.own_hi + uw
        for sweeps, width, zlo, zhi, slo, shi in blocks:
            assert plo <= zlo and zhi <= phi and 0 <= width <= halo and 0 <= sweeps <= halo
        ranks.append(dict(d=d, div=ldiv, solid=lsolid, nbr=lnbr, bufs=[np.zeros_like(ldiv), np.zeros_like(ldiv)],
                          blocks=blocks))
    done = 0
    for b in range(nblk):
        width = scheds[0][1][b][1]
        assert all(s[1][b][1] == width for s in scheds)
        if width:
            cur = [q["bufs"][done & 1] for q in ranks]
            for lo, hi in zip(range(world - 1), range(1, world)):
                a, c = ranks[lo]["d"], ranks[hi]["d"]
                cur[hi][c.own_lo - width:c.own_lo] = cur[lo][a.own_hi - width:a.own_hi]
                cur[lo][a.own_hi:a.own_hi + width] = cur[hi][c.own_lo:c.own_lo + width]
            for q, t in zip(ranks, cur):          # ghost planes beyond the exchange hold stale values: poison them
                d = q["d"]
                if d.rank > 0:
                    t[:d.own_lo - width] = np.nan
                if d.rank < world - 1:
                    t[d.own_hi + width:] = np.nan
        sweeps = scheds[0][1][b][0]
        for q in ranks:
            _, _, zlo, zhi, slo, shi = q["blocks"][b]
            for s in range(sweeps):
                _sweep(q["bufs"][(done + s) & 1], q["bufs"][(done + s + 1) & 1], q["div"], q["solid"], q["nbr"],
                       zlo + s * slo, zhi - s * shi)
        done += sweeps
    assert done == iters
    return [(q["d"], q["bufs"][done & 1]) for q in ranks]


CASES = [(world, margin, gnz, iters)
         for world, margin, gnz in [(2, 2, 12), (2, 2, 17), (3, 2, 20), (4, 2, 24), (4, 2, 27), (2, 3, 16), (3, 3, 25),
                                    (4, 3, 35)]
         for iters in sorted({1, 2 * margin + 1, 2 * margin + 2, 2 * margin + 3, 2 * (2 * margin + 2), 34})]


@pytest.mark.parametrize("world,margin,gnz,iters", CASES)
def test_schedule_reproduces_the_undivided_sweeps(world, margin, gnz, iters):
    solid, nbr, div = _problem(gnz, 6, 7, seed=gnz * 100 + world * 10 + margin)
    want = _undivided(solid, nbr, div, iters)
    for d, p in _slabbed(solid, nbr, div, world, margin, iters):
        got = p[d.own_lo - (1 if d.rank > 0 else 0):d.own_hi]
        ref = want[d.z0 - (1 if d.rank > 0 else 0):d.z1]
        assert np.array_equal(got, ref), "rank %d" % d.rank


@pytest.mark.parametrize("world,margin,iters", [(2, 2, 1), (2, 2, 6), (3, 3, 100), (4, 2, 100)])
def test_schedule_shape(world, margin, iters):
    halo = 2 * margin + 2
    gnz = world * halo + 1
    for r in range(world):
        (plo, phi, uw), blocks = jacobi_schedule(gnz, world, r, margin, iters)
        assert len(blocks) == -(-(iters + 1) // halo)
        assert sum(b[0] for b in blocks) == iters
        assert blocks[0][1] == 0 and all(b[1] > 0 for b in blocks[1:])
        assert all(b[0] == halo for b in blocks[:-1]) and blocks[-1][0] <= halo - 1
        assert 1 <= uw <= halo
    (plo, phi, uw), blocks = jacobi_schedule(gnz, 1, 0, margin, iters)
    assert blocks == [(iters, 0, 0, gnz, 0, 0)] and (plo, phi, uw) == (0, gnz, 0)


@pytest.mark.parametrize("args", [(24, 2, 0, 2, 0), (24, 2, 0, 1, 10), (10, 2, 0, 2, 10), (24, 2, 2, 2, 10),
                                  (2, 1, 0, 2, 10)])
def test_schedule_refusals(args):
    with pytest.raises(ValueError):
        jacobi_schedule(*args)
