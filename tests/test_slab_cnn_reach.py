"""How far across a rank boundary the banked projection network reaches, checked without a GPU: the smallest z-slab
margin of a model with N banks (tfl_slab_cnn_margin) must give a halo (2 margin + 2 ghost planes) that holds every
plane that can change the projection's output on the owned planes, and the U / p exchange before the projection
(2 margin + 1 planes) every plane of U or p that can; one margin less must not do, at the worst alignment of the
rank's boundary to the coarsest bank's 2^(N-1) planes.

The model is a float64 restatement of the step's projection on the 3-D 'default' graph with banks split at stage 1
and joined at stage 3 (oracle/model.py's 'mres' graph, lib/model.lua:252-361): wall mask, divergence and occupancy in
front, the velocity update and wall mask behind.  Its dependency structure follows the kernels (the input at plane z
reads U at z and z + 1 and the flags at z - 1 .. z + 1; the update at z reads p and the flags at z - 1).  The input
scale is a global reduction the slab step all-reduces, not a halo matter: it is held fixed.  Weights are positive
and biases large, so every ReLU passes and no influence is hidden.  One plane of U, p or flags at a time is
perturbed and the output planes that change are recorded."""
import pytest
import torch
import torch.nn.functional as F

from fluidnet_b200.slab import cnn_margin

FLUID, OBST, EMPTY = 1, 2, 4


def _prev(t, dim):
    """t at index - 1 along dim (index 0 gets 0: no neighbour)."""
    out = torch.roll(t, 1, dim)
    out.select(dim, 0).zero_()
    return out


def _wall_zero(flags):
    """[3][Z][Y][X] bool: component a of U is zeroed (wall_bc_zero_mask)."""
    cf, co = (flags & FLUID) != 0, (flags & OBST) != 0
    zs = []
    for dim in (2, 1, 0):                     # x, y, z components: neighbour at index - 1
        nb = _prev(flags, dim)
        has = torch.ones_like(cf)
        has.select(dim, 0).zero_()
        zs.append((cf | co) & has & (((nb & OBST) != 0) | (co & ((nb & FLUID) != 0))))
    return torch.stack(zs)


def _border(shape):
    z, y, x = shape
    b = torch.zeros(shape, dtype=torch.bool)
    b[0], b[-1], b[:, 0], b[:, -1], b[:, :, 0], b[:, :, -1] = True, True, True, True, True, True
    return b


def _net(x, w, n, add):
    hl = [x[None]]
    for _ in range(1, n):
        hl.append(F.avg_pool3d(hl[-1], 2))
    outs = []
    for i, h in enumerate(hl):
        h = F.relu(F.conv3d(h, w["l1"][i], w["b1"][i], padding=1))
        h = F.relu(F.conv3d(h, w["l2"][i], w["b2"][i], padding=1))
        outs.append(F.interpolate(h, scale_factor=2 ** i, mode="nearest") if i else h)
    h = sum(outs[1:], outs[0]) if add else torch.cat(outs, 1)
    h = F.relu(F.conv3d(h, w["l3"], w["b3"], padding=1))
    h = F.relu(F.conv3d(h, w["l4"], w["b4"]))
    return F.conv3d(h, w["l5"], w["b5"])[0, 0]


def project(U, p, flags, w, n, add):
    """The slab step's projection with scale 1: (p, U) after the network and the velocity update."""
    border = _border(flags.shape)
    fluid = (flags & FLUID) != 0
    U1 = torch.where(_wall_zero(flags), torch.zeros_like(U), U)
    nxt = lambda t, dim: torch.roll(t, -1, dim)
    dv = (U1[0] - nxt(U1[0], 2)) + (U1[1] - nxt(U1[1], 1)) + (U1[2] - nxt(U1[2], 0))
    dv = torch.where(fluid & ~border, dv, torch.zeros_like(dv))
    occ = torch.where(flags == FLUID, 0.0, torch.where(flags == OBST, 1.0, -1.0)).double()
    pn = _net(torch.stack([p, dv, occ]), w, n, add)
    u = U1.clone()
    for a, dim in enumerate((2, 1, 0)):
        fn, pp = _prev(flags, dim), _prev(pn, dim)
        upd = torch.where((fn & FLUID) != 0, u[a] - (pn - pp), u[a])
        upd = torch.where((fn & EMPTY) != 0, upd - pn, upd)
        u[a] = torch.where(fluid & ~border, upd, u[a])
    u = torch.where(_wall_zero(flags), torch.zeros_like(u), u)
    return pn, u


def _weights(n, add, gen):
    r = lambda *s: torch.rand(*s, generator=gen, dtype=torch.float64)
    return {"l1": [r(8, 3, 3, 3, 3) * 0.1 for _ in range(n)], "b1": [r(8) + 4.0 for _ in range(n)],
            "l2": [r(8, 8, 3, 3, 3) * 0.05 for _ in range(n)], "b2": [r(8) + 1.0 for _ in range(n)],
            "l3": r(8, 8 if add else 8 * n, 3, 3, 3) * 0.05, "b3": r(8) + 1.0,
            "l4": r(8, 8, 1, 1, 1) * 0.2, "b4": r(8) + 1.0, "l5": r(1, 8, 1, 1, 1), "b5": r(1)}


def _influence(n, add, nz=128):
    """{field: [set of output planes that change when plane q of the field is perturbed, per q]}."""
    gen = torch.Generator().manual_seed(n)
    ny = nx = max(8, 2 ** (n - 1))
    shape = (nz, ny, nx)
    flags = torch.full(shape, FLUID, dtype=torch.int32)
    flags[_border(shape)] = OBST
    U = torch.rand((3,) + shape, generator=gen, dtype=torch.float64) - 0.5
    p = torch.rand(shape, generator=gen, dtype=torch.float64)
    w = _weights(n, add, gen)
    base_p, base_u = project(U, p, flags, w, n, add)
    tol = 1e-12 * max(base_p.abs().max().item(), base_u.abs().max().item())
    out = {"U": [], "p": [], "flags": []}
    for q in range(nz):
        for field in out:
            u2, p2, f2 = U.clone(), p.clone(), flags.clone()
            if field == "U":
                u2[:, q] += 0.25
            elif field == "p":
                p2[q] += 0.25
            else:
                f2[q, 1:-1:2, 1:-1:3] = OBST
            gp, gu = project(u2, p2, f2, w, n, add)
            changed = ((gp - base_p).abs() > tol) | ((gu - base_u).abs() > tol).any(0)
            out[field].append(set(changed.reshape(nz, -1).any(1).nonzero().flatten().tolist()))
    return out


def _reach(infl, fields, z0, z1):
    """Farthest plane below z0 (distance z0 - q) and above z1 - 1 (q - z1 + 1) whose perturbation changes an
    output on the owned planes [z0, z1)."""
    lo = hi = 0
    for f in fields:
        for q, planes in enumerate(infl[f]):
            if not any(z0 <= z < z1 for z in planes):
                continue
            if q < z0:
                lo = max(lo, z0 - q)
            if q >= z1:
                hi = max(hi, q - z1 + 1)
    return lo, hi


@pytest.mark.parametrize("agg", ["concat", "add"])
@pytest.mark.parametrize("n", [1, 2, 3, 4, 5])
def test_margin_holds_the_reach_and_is_tight(n, agg):
    s = 2 ** (n - 1)
    margin = cnn_margin(n)
    if n == 1:
        assert margin == 2
    infl = _influence(n, agg == "add")
    worst = worst_uv = 0
    center = 56                  # every cone stays clear of the global ends of the 128 planes
    for a in range(s):           # the owned boundary at every residue mod s; one owned plane suffices
        z = center + a
        lo, hi = _reach(infl, ("U", "p", "flags"), z, z + 1)
        lo_uv, hi_uv = _reach(infl, ("U", "p"), z, z + 1)
        assert max(lo, hi) <= 2 * margin + 2, (a, lo, hi)
        assert max(lo_uv, hi_uv) <= 2 * margin + 1, (a, lo_uv, hi_uv)
        worst, worst_uv = max(worst, lo, hi), max(worst_uv, lo_uv, hi_uv)
    # one margin less does not hold the worst alignment's reach
    assert worst > 2 * (margin - 1) + 2, (worst, margin)
    if n > 1:
        assert worst == 3 * s + 2 and worst_uv == 3 * s + 1, (worst, worst_uv)


def test_margin_of_the_supported_bank_counts():
    assert [cnn_margin(n) for n in range(0, 9)] == [2, 2, 3, 6, 12, 24, 48, 96, 192]
    with pytest.raises(ValueError):
        cnn_margin(9)
