"""Lattice advection inputs, shared by tests/test_oracle_lattice.py (oracle vs the compiled reference) and
tests/test_gpu_lattice.py (kernels vs the oracle).

Random velocities almost never put a trace on the boundary of a comparison that picks a branch.  These do, on purpose:
  - velocities are axis-aligned.  In each field only one component is non-zero, constant along each row of that axis
    (in 3-D only every other row in both perpendicular directions carries a value).  So a cell's centred velocity and the
    velocity at its face of that axis are (u, 0, 0) exactly, the other two face traces are u / 2 long, and the
    displacement u * dt is exact in fp32: sqrt(d^2) = |d| and the trace direction is +-1 exactly.
  - u is searched among the floats near target / dt so that float32(u) * float32(dt) equals the target length
    exactly (numpy's float32 multiply is IEEE's).  Targets: 0.25 k up to 3 cells (cell faces, centres, neighbour
    centres, the domain ends, the faces of solids) and one ulp either side of them, and the branch thresholds of the
    trace loop and the clear-space fast paths (tfl_device.cuh, tfl_advect_tile.cu) with +-1 and +-2 ulps.
  - dt is 0.25, 0.1 or 0.3.
tie_census counts, in numpy, the cells whose traces end exactly on a centre, a face, a domain end or the face of a
solid, and the cells whose trace length equals each threshold, so the tests can hold the inputs to minimum counts."""
import functools

import numpy as np

from fluidnet_b200 import synth

F32 = np.float32
K_CLEAR_MAX = 7                     # tfl_device.cuh: clearance is capped at kClearMax + 1
HIT_MARGIN = F32(1e-5)              # TFL_HIT_MARGIN: line_trace's loop runs while travelled < length - 1e-5
DTS = (0.25, 0.1, 0.3)
DIMS3 = (40, 24, 20)                # x a multiple of 4 (the tile kernels' TMA rows), not of the 32-cell tile
DIMS2 = (40, 36, 1)
FLAG_KINDS = ("box", "open", "geom", "exotic")


def clear_reach(clr):
    """tfl_device.cuh clear_reach: (float)clr - (0.5f + TFL_CLEAR_SLACK)."""
    return F32(clr) - (F32(0.5) + F32(0.01))


def clear_reach_fluid(clr):
    return F32(clr) - (F32(1.0) + F32(0.01))


def tile_reach(hf):
    """The tile kernels' REACH = (float)HF - 0.51f."""
    return F32(hf) - F32(0.51)


def ulps(x, n):
    x = F32(x)
    for _ in range(abs(n)):
        x = np.nextafter(x, F32(np.inf) if n > 0 else F32(-np.inf), dtype=np.float32)
    return F32(x)


def thresholds():
    """name -> float32 length of every branch threshold on the trace length."""
    t = {"halo1": tile_reach(1), "halo2": tile_reach(2)}
    for c in range(1, K_CLEAR_MAX + 2):
        t["reach%d" % c] = clear_reach(c)
        if c >= 2:
            t["reach_fluid%d" % c] = clear_reach_fluid(c)
    for k in range(4):
        t["step%d" % k] = F32(k) + HIT_MARGIN
    return t


def target_lengths():
    """Every target trace length (float32, positive, sorted, distinct)."""
    out = set()
    for k in range(1, 13):
        for n in (-1, 0, 1):
            out.add(float(ulps(0.25 * k, n)))
    for v in thresholds().values():
        for n in (-2, -1, 0, 1, 2):
            x = ulps(v, n)
            if x > 0:
                out.add(float(x))
    return [F32(x) for x in sorted(out)]


@functools.lru_cache(maxsize=None)
def speeds(dt):
    """Every target length reachable at dt, with its speed: [(length, u)]."""
    out = [(L, speed_for(L, dt)) for L in target_lengths()]
    return [(L, u) for L, u in out if u is not None]


def speed_for(length, dt):
    """A float32 u with float32(u) * float32(dt) == length whose MAC average 0.25 * (((u + u) + u) + u) is u again, or
    None (then some products skip that length)."""
    length, dt = F32(length), F32(dt)
    u0 = F32(float(length) / float(dt))
    cands = [u0]
    up = down = u0
    for _ in range(256):
        up = np.nextafter(up, F32(np.inf), dtype=np.float32)
        down = np.nextafter(down, F32(0), dtype=np.float32)
        cands += [up, down]
    for u in cands:
        if F32(u * dt) == length and F32(F32(0.25) * F32(F32(F32(u + u) + u) + u)) == u:
            return F32(u)
    return None


def make_flags(kind, is3d, nb=1):
    nx, ny, nz = DIMS3 if is3d else DIMS2
    if kind == "open":
        # fluid everywhere, border included: traces can reach the domain ends
        return np.ascontiguousarray(np.full((nb, 1, nz, ny, nx), synth.FLUID, np.float32))
    return synth.make_flags(nx, ny, nz, is3d, nb=nb, geometry=kind != "box", exotic=kind == "exotic")


def make_velocity(flags, is3d, axis, dt, offset=0, max_length=None):
    """One non-zero component (axis), constant along each row of that axis; in 3-D the rows at even perpendicular
    indices carry a target length (with a sign that alternates) and the others are 0, so that the two other face
    traces of a cell are at most half as long (the tile kernels test the longest of the three); in 2-D every row
    does.  Row r takes target (r * 7 + offset) mod L, among the targets up to max_length cells if given."""
    nb, _, nz, ny, nx = flags.shape
    nc = 3 if is3d else 2
    U = np.zeros((nb, nc, nz, ny, nx), np.float32)
    us = [u for L, u in speeds(dt) if max_length is None or L <= max_length]
    every = 2 if is3d else 1
    ext = (nx, ny, nz)
    perp = [a for a in range(nc) if a != axis]
    r = 0
    for b in range(nb):
        grids = [range(0, ext[a], every) for a in perp]
        idx = [(p, q) for p in grids[0] for q in (grids[1] if len(grids) > 1 else [0])]
        for p, q in idx:
            u = us[(r * 7 + offset + 13 * b) % len(us)]
            s = F32(1.0) if (r // 2) % 2 == 0 else F32(-1.0)
            sl = [slice(None)] * 3                          # (z, y, x)
            sl[2 - perp[0]] = p
            if len(perp) > 1:
                sl[2 - perp[1]] = q
            elif not is3d:
                sl[0] = 0
            U[b, axis][tuple(sl)] = s * u
            r += 1
    return np.ascontiguousarray(U)


def density(flags):
    """Density on a 1/64 lattice with zeros (zero clamp bounds), 0 outside fluid."""
    rs = np.random.RandomState(11)
    d = (rs.randint(0, 65, size=flags.shape) / 64.0).astype(np.float32)
    d[rs.rand(*flags.shape) < 0.3] = 0.0
    d[(flags.astype(np.int32) & 1) == 0] = 0.0
    return np.ascontiguousarray(d)


# (name, is3d, flag kind, axis, dt)
FIELD_CASES = [("%s_%s_ax%d_dt%g" % ("3d" if is3d else "2d", kind, axis, dt), is3d, kind, axis, dt)
               for is3d in (True, False) for kind in FLAG_KINDS for axis in range(3 if is3d else 2) for dt in DTS]
FIELD_IDS = [c[0] for c in FIELD_CASES]


def build(case, nb=1, wall_bcs=None):
    """flags, U (wall BCs applied by wall_bcs(U, flags) if given), density."""
    name, is3d, kind, axis, dt = case
    flags = make_flags(kind, is3d, nb)
    U = make_velocity(flags, is3d, axis, dt, offset=FIELD_CASES.index(case))
    if wall_bcs is not None:
        wall_bcs(U, flags)
    return dict(name=name, is3d=is3d, dt=dt, flags=flags, U=U, density=density(flags))


def clearance(flags, is3d):
    """The clearance field of launch_clearance (tfl_stencils.cu): 0 for cells that are not fluid or lie on an end of
    the storage, else 1 + the largest r <= kClearMax whose (2r+1)^2 or ^3 box is all such usable cells."""
    from scipy import ndimage
    fl = flags[:, 0].astype(np.int32)
    nb, nz, ny, nx = fl.shape
    usable = (fl & 1) != 0
    usable[:, :, :, 0] = usable[:, :, :, -1] = False
    usable[:, :, 0, :] = usable[:, :, -1, :] = False
    if is3d:
        usable[:, 0] = usable[:, -1] = False
    clr = np.where(usable, 1, 0).astype(np.int32)
    for r in range(1, K_CLEAR_MAX + 1):
        size = (1, 2 * r + 1 if is3d else 1, 2 * r + 1, 2 * r + 1)
        box = ndimage.minimum_filter(usable.astype(np.uint8), size=size, mode="constant", cval=0).astype(bool)
        clr[box] = r + 1
    return clr


def tie_census(flags, U, dt):
    """Counts over the fluid cells of every batch entry and both trace directions (the forward trace -u dt and the
    backward +u dt of MacCormack) of the centred velocity: traces that end exactly on a cell centre, a cell face, a
    domain end, or the face of a non-fluid cell; and traces whose length equals each threshold (keys of thresholds(),
    the clearance ones only at cells of that clearance, 'reach' / 'reach_fluid' summing them)."""
    is3d = U.shape[1] == 3
    nb, nc, nz, ny, nx = U.shape
    dt = F32(dt)
    fl = flags[:, 0].astype(np.int32)
    fluid = (fl & 1) != 0
    clr = clearance(flags, is3d)
    cen = []
    for a in range(nc):
        u = U[:, a]
        nxt = np.zeros_like(u)
        if a == 0:
            nxt[..., :-1] = u[..., 1:]
        elif a == 1:
            nxt[..., :-1, :] = u[..., 1:, :]
        else:
            nxt[:, :-1] = u[:, 1:]
        cen.append(F32(0.5) * (u + nxt))
    cen = np.stack(cen, 1).astype(np.float32)
    counts = dict.fromkeys(("centre", "face", "domain_end", "solid_face"), 0)
    th = thresholds()
    counts.update(dict.fromkeys(th, 0))
    counts["reach"] = counts["reach_fluid"] = 0
    ext = (nx, ny, nz)
    nonzero = (cen != 0).sum(1)
    for a in range(nc):
        moving = fluid & (nonzero == 1) & (cen[:, a] != 0)
        bb, kk, jj, ii = np.nonzero(moving)
        start = np.stack([ii, jj, kk], 1).astype(np.float64) + 0.5
        for sgn in (F32(-1.0), F32(1.0)):
            d = (cen[bb, a, kk, jj, ii] * (sgn * dt)).astype(np.float32)
            length = np.abs(d)
            end = start[:, a] + d.astype(np.float64)
            frac = end - np.floor(end)
            on_face = (frac == 0) & (end > 0) & (end < ext[a])
            counts["centre"] += int((frac == 0.5).sum())
            counts["face"] += int(on_face.sum())
            counts["domain_end"] += int(((end == 0) | (end == ext[a])).sum())
            beyond = np.where(d > 0, end, end - 1).astype(np.int64)
            idx = [bb, kk, jj, ii]
            sel = np.nonzero(on_face)[0]
            pos = [x[sel].copy() for x in idx]
            pos[3 - a] = beyond[sel]
            counts["solid_face"] += int((~fluid[tuple(pos)]).sum())
            c = clr[bb, kk, jj, ii]
            for name, v in th.items():
                if name.startswith("reach_fluid"):
                    hit = (length == v) & (c == int(name[11:]))
                    counts["reach_fluid"] += int(hit.sum())
                elif name.startswith("reach"):
                    hit = (length == v) & (c == int(name[5:]))
                    counts["reach"] += int(hit.sum())
                else:
                    hit = length == v
                counts[name] += int(hit.sum())
    return counts


def trace_starts(flags, is3d, cells=50):
    """(pos, delta) pairs for calcLineTrace: the centres of `cells` fluid cells, evenly spread over those within two
    cells of a solid or an end of the storage, each with axis-aligned deltas 0.25 k (k = 1 .. 12) along one axis and
    direction (taken in turn), which end on faces, centres, the domain ends and the faces of solids."""
    fl = flags[0, 0].astype(np.int32)
    clr = clearance(flags, is3d)[0]
    kk, jj, ii = np.nonzero(((fl & 1) != 0) & (clr <= 2))
    pick = np.linspace(0, len(kk) - 1, cells).round().astype(int)
    out = []
    for n, c in enumerate(pick):
        k, j, i = kk[c], jj[c], ii[c]
        pos = np.array([i + 0.5, j + 0.5, k + 0.5 if is3d else 0.5], np.float32)
        a, s = (n // 2) % (3 if is3d else 2), (-1.0, 1.0)[n % 2]
        for step in range(1, 13):
            d = np.zeros(3, np.float32)
            d[a] = F32(s * 0.25 * step)
            out.append((pos, d))
    return out
