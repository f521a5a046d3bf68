"""The z-slab convnet step (tfl_cnn_stats on each rank, the all-reduce of the two sums, tfl_cnn_project_from_sums)
against float64 per voxel, and its projection held to the planes DESIGN.md ("Banked models on slabs") says it reads.

Emulated ranks on one GPU (SlabSimulator.phases() driven by `lockstep`, run_lockstep with hooks), three steps per
case, each referenced from the gathered slab state before it:

  * At the ("sum", ...) request: the owned planes of every rank's U1, gathered, equal bit for bit the U1 of the
    whole-grid operator sequence from the same state (network_bound.input_fields), so a difference before the
    projection is never blamed on the network.  Each rank's partial (sum, sum of squares) lies within the
    double-summation bound gamma53_(n-1) sum |x| of the exact sums over its owned planes (the kernel adds n float
    terms in double in an order of its own), and the scale from the rank-order total lies in the scale_interval the
    float64 bound is built on.
  * Reach: before tfl_cnn_project_from_sums every rank's planes outside the documented reach are poisoned -- U1 and
    pDiv with a quiet NaN, the flags all obstacle in one run and all fluid in another -- and p and U must equal an
    unpoisoned twin call bit for bit; the poisoned planes are restored before the step goes on.  The reach, local
    planes, for the coarsest bank scale s = 2^(N-1): pDiv [own_lo - 3s - 1, own_hi + 3s), U1 one plane further up,
    the flags one plane further down (tests/test_slab_cnn_reach.py pins these numbers on a float64 model).
  * Writes: around the twin call, p and U outside the owned planes, U1 and the flags keep their bits.  The velocity
    update of plane own_lo reads the network's p on own_lo - 1, but that value stays in the call's scratch: p's
    ghost planes are not written (the next step's first exchange refreshes them), so p on own_lo - 1 is pinned here
    rather than compared with float64; it enters U's z component on own_lo, which is.
  * After the step: the gathered p and U within the bound E of tests/network_bound.py at every voxel, the reference
    being projection_reference (tests/network_bound.py) on the gathered start state with a whole-grid model
    in the same mode; after step 1 the density is bit-exact.  Each case prints its largest err / E and the largest per
    distance from the nearest rank boundary (0: the two planes either side of it).

Cases (CASES, checked without a GPU by test_case_table_reaches_every_edge): worlds 2, 3 and 4; N = 1, N = 2 and 3
('concat' and 'add'), each in 3xTF32 and TF32; for N = 3 a rank boundary at every residue mod 4, uneven slabs, the
thinnest legal slab (slab = halo) and a margin above the minimum.  In every case the plume's inflow cylinder straddles
the first rank boundary; with three or more ranks the last one runs through slow fluid (|U| below 1e-2 of its
maximum on every plane of U within reach, on the start state).  The world-1 library driver (NativeSlabSimulator)
gets the per-voxel check too.

Largest err / E measured on an H100 80GB HBM3 (SXM, 700 W power limit), p / U: 3xTF32 0.043 / 0.18, TF32
0.067 / 0.0017, the world-1 library driver 0.027 / 0.13; no trend with the distance from a boundary.  The file runs
in about 15 s.

Faults injected once each, not kept:
  * The phase-2 U / p exchange one plane narrower (slab.py): the per-voxel check fails at N = 2 in 3xTF32, where the
    boundaries sit on even planes, the worst alignment for s = 2 (p, err / E up to 2.0 in step 1).  The other cases
    stay within their bounds: a single bank has one plane of slack (reach 4, exchange 5), TF32 bounds are 2^8 wider,
    and at N = 3 the stale plane's one-step change stays below E.  test_gpu_slab_banks.py and test_gpu_slab_ranks.py
    fail too.
  * The velocity update one plane further down on an interior side (reads p_net, U1 and the flags of one more plane,
    writes p and U on own_lo - 1): the writes check fails in every multi-rank case; no earlier test fails.
  * The convolution stack computing p_net one plane further down (so reading the network input one plane further):
    nothing fails, and nothing can through p and U -- the extra plane of p_net is never read by the velocity update,
    so every output bit stays, NaN beyond the reach included.
  * tfl_cnn_stats summing one ghost plane: the partial-sum check fails in every multi-rank case; so do the emulated
    cases of test_gpu_slab.py, test_gpu_slab_banks.py and test_gpu_cnn_network_f64.py and test_gpu_slab_ranks.py."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import oracle
from fluidnet_b200 import synth
from network_bound import U64, check, input_fields, projection_reference, scale_interval
from scenes import banks, plume_batch, step_mconf

FLUID, OBSTACLE = 1.0, 2.0
SLOW = 1e-3                 # U's factor on the slow boundary's planes
BC_KEYS = ("UBC", "UBCInvMask", "densityBC", "densityBCInvMask")

# (world, gnz, ny, nx, banksNum, aggregate, mode, margin or None: the model's minimum)
CASES = [
    (2, 24, 16, 16, 1, None, "tf32x3", None),
    (3, 20, 16, 16, 1, None, "tf32", None),          # uneven: 7, 7, 6
    (4, 24, 16, 16, 1, None, "tf32x3", None),        # slab 6 = halo 6
    (2, 32, 16, 16, 2, "concat", "tf32x3", None),
    (3, 46, 16, 24, 2, "concat", "tf32", None),      # uneven: 16, 15, 15
    (4, 32, 16, 16, 2, "add", "tf32x3", None),       # slab 8 = halo 8
    (3, 42, 16, 16, 2, "add", "tf32", 4),            # margin above the minimum
    (2, 28, 16, 16, 3, "add", "tf32", None),         # slab 14 = halo 14; boundary 14 = 2 mod 4
    (3, 56, 16, 16, 3, "concat", "tf32x3", None),    # uneven: 19, 19, 18; boundaries 3, 2 mod 4
    (4, 60, 16, 16, 3, "concat", "tf32", None),      # boundaries 3, 2, 1 mod 4
    (3, 48, 16, 16, 3, "add", "tf32x3", 7),          # margin above the minimum, slab 16 = halo 16; 0 mod 4
]


def case_id(c):
    return "w%d-%dx%dx%d-N%d-%s-%s-m%s" % c


def decompositions(case):
    from fluidnet_b200.slab import SlabDecomposition, cnn_margin
    world, gnz, n, margin = case[0], case[1], case[4], case[7]
    m = margin or cnn_margin(n)
    return [SlabDecomposition(gnz, r, world, 2 * m + 2) for r in range(world)], m


def boundaries(case):
    """Global plane z0 of every rank but the first."""
    return [d.z0 for d in decompositions(case)[0][1:]]


def reach(n):
    """Planes below own_lo and from own_hi on that the projection may read, per field: {field: (below, above)}."""
    s = 2 ** (n - 1)
    return {"pDiv": (3 * s + 1, 3 * s), "U1": (3 * s + 1, 3 * s + 1), "flags": (3 * s + 2, 3 * s)}


def plume_and_slow(case):
    """(the boundary the plume straddles, the boundary through slow fluid or None)."""
    b = boundaries(case)
    if not b:
        return max(case[1] // 2, 1) - 1, None
    return b[0], (b[-1] if len(b) > 1 else None)


def problem(case):
    """Global CPU tensors of the start state, mconf, the model's numpy weights and its banks."""
    world, gnz, ny, nx, n, agg, mode, margin = case
    batch = plume_batch((gnz, ny, nx), inflow=nx / 128.0 * 4)
    plume, slow = plume_and_slow(case)
    if slow is not None:
        lo, hi = reach(n)["U1"]
        batch["UDiv"][:, :, slow - lo:slow + hi] *= np.float32(SLOW)
    batch["pDiv"] = ((np.random.RandomState(gnz).rand(*batch["flags"].shape) - 0.5) * 0.2).astype(np.float32)
    # the inflow cylinder is centred on plane max(gnz // 2, 1) - 1; it is z-invariant elsewhere, so a roll moves it
    shift = plume - (max(gnz // 2, 1) - 1)
    for k in BC_KEYS:
        batch[k] = np.ascontiguousarray(np.roll(batch[k], shift, axis=2))
    bk = None if n == 1 else banks(n, agg)
    return {k: torch.from_numpy(v) for k, v in batch.items()}, step_mconf(nx), synth.make_model(True, banks=bk), bk


def test_case_table_reaches_every_edge():
    """The table covers what the docstring promises, and each case's start state has its plume and slow boundary."""
    from fluidnet_b200.slab import cnn_margin
    assert {c[0] for c in CASES} == {2, 3, 4}
    assert {(c[4], c[5], c[6]) for c in CASES} == {(1, None, m) for m in ("tf32x3", "tf32")} | {
        (n, a, m) for n in (2, 3) for a in ("concat", "add") for m in ("tf32x3", "tf32")}
    n3 = [c for c in CASES if c[4] == 3]
    assert {b % 4 for c in n3 for b in boundaries(c)} == {0, 1, 2, 3}
    sizes = lambda c: [d.z1 - d.z0 for d in decompositions(c)[0]]
    assert any(len(set(sizes(c))) > 1 for c in n3)
    assert any(min(sizes(c)) == decompositions(c)[0][0].halo for c in n3)
    assert any(c[7] is not None and c[7] > cnn_margin(c[4]) for c in n3)
    for c in CASES:
        world, gnz, ny, nx, n = c[:5]
        decs, m = decompositions(c)
        assert m >= cnn_margin(n) and gnz % 2 ** (n - 1) == 0 and nx % 2 ** (n - 1) == 0 and ny % 2 ** (n - 1) == 0
        assert min(sizes(c)) >= decs[0].halo
        tb, _, _, _ = problem(c)
        plume, slow = plume_and_slow(c)
        inflow = (tb["UBC"][0, 1] != 0).flatten(1).any(1)
        assert inflow[plume - 1] and inflow[plume], (c, "the plume does not cross its boundary")
        assert (slow is not None) == (world >= 3), c
        if slow is not None:
            Us = tb["UDiv"] * tb["UBCInvMask"] + tb["UBC"]
            lo, hi = reach(n)["U1"]
            for u in (tb["UDiv"], Us):
                near = u[:, :, slow - lo:slow + hi].abs().max().item()
                assert near < 1e-2 * u.abs().max().item(), (c, near, u.abs().max().item())
            assert not inflow[slow - lo:slow + hi].any(), c


# ---------------------------------------------------------------------------------------------------------------
# The emulated ranks
# ---------------------------------------------------------------------------------------------------------------
def lockstep(sims, on_sums=None, on_project=None):
    """slab.run_lockstep with two hooks around the sum request: on_sums(sims) sees every rank's partial sums and U1
    before the reduction, on_project(sims) runs after it, before any rank resumes into tfl_cnn_project_from_sums."""
    sims = sorted(sims, key=lambda q: q.dec.rank)
    gens = [q.phases() for q in sims]
    while True:
        reqs = []
        for g in gens:
            try:
                reqs.append(next(g))
            except StopIteration:
                reqs.append(None)
        if all(r is None for r in reqs):
            return
        assert all(r is not None for r in reqs) and len({r[0] for r in reqs}) == 1
        if reqs[0][0] == "sum":
            if on_sums:
                on_sums(sims)
            total = sum(r[1].clone() for r in reqs)
            for r in reqs:
                r[1].copy_(total)
            if on_project:
                on_project(sims)
        else:
            width = reqs[0][2]
            for lo, hi in zip(range(len(sims) - 1), range(1, len(sims))):
                a, b = sims[lo].dec, sims[hi].dec
                for ta, tb in zip(reqs[lo][1], reqs[hi][1]):
                    tb[:, :, b.own_lo - width:b.own_lo].copy_(ta[:, :, a.own_hi - width:a.own_hi])
                    ta[:, :, a.own_hi:a.own_hi + width].copy_(tb[:, :, b.own_lo:b.own_lo + width])


def project(q):
    """The slab step's tfl_cnn_project_from_sums call, on q's current arrays and sums."""
    t, c, d, s = q.tfluids, q.ctx, q.dec, q.s
    with q._slab(d.own_lo, d.own_hi):
        c.use_current_stream()
        c.check(c.lib.tfl_cnn_project_from_sums(c.h, q.model.h, t._grid(s["pDiv"]), t._grid(q.U1), t._grid(s["flags"]),
                                                C.c_void_p(q.sums.data_ptr()), t._grid(s["pDiv"]), t._grid(s["UDiv"]),
                                                float(q.model.threshold)))
    torch.cuda.synchronize()


def bits(t):
    return t.contiguous().view(torch.int32)


def same_bits(a, b):
    return torch.equal(bits(a), bits(b))


def outside(d, lo, hi):
    """Local plane slices outside [own_lo - lo, own_hi + hi) on the sides with a neighbour."""
    out = []
    if d.lo_halo and d.own_lo - lo > 0:
        out.append(slice(0, d.own_lo - lo))
    if d.hi_halo and d.own_hi + hi < d.nz:
        out.append(slice(d.own_hi + hi, d.nz))
    return out


def check_writes_and_reach(q, n, what):
    """The twin call, the writes around it and the two poisoned calls against it.  Leaves every array as it was."""
    d, s = q.dec, q.s
    arrays = {"pDiv": s["pDiv"], "UDiv": s["UDiv"], "U1": q.U1, "flags": s["flags"]}
    keep = {k: v.clone() for k, v in arrays.items()}

    def restore():
        for k, v in arrays.items():
            v.copy_(keep[k])

    project(q)
    twin = {k: arrays[k].clone() for k in ("pDiv", "UDiv")}
    for k in ("pDiv", "UDiv"):
        for sl in outside(d, 0, 0):
            assert same_bits(arrays[k][:, :, sl], keep[k][:, :, sl]), "%s: %s written on planes %s" % (what, k, sl)
    for k in ("U1", "flags"):
        assert same_bits(arrays[k], keep[k]), "%s: the projection wrote its input %s" % (what, k)
    restore()
    own = slice(d.own_lo, d.own_hi)
    for code in (OBSTACLE, FLUID):
        for k, (lo, hi) in reach(n).items():
            for sl in outside(d, lo, hi):
                arrays[k][:, :, sl] = code if k == "flags" else float("nan")
        project(q)
        for k in ("pDiv", "UDiv"):
            assert same_bits(arrays[k][:, :, own], twin[k][:, :, own]), (
                "%s: %s differs once the planes beyond the documented reach hold %s" % (
                    what, k, "obstacle flags and NaN" if code == OBSTACLE else "fluid flags and NaN"))
        restore()
    return twin["pDiv"][:, :, own]


def gather(sims, key):
    return torch.cat([q.dec.owned(q.s[key]).cpu() for q in sims], dim=2)


def pre_projection(state, mconf, gm):
    """The whole-grid operator sequence up to the projection from `state` (GPU tensors, left as they are)."""
    from fluidnet_b200 import simulate
    ob = {k: v.clone() for k, v in state.items()}
    simulate.simulate(None, mconf, ob, gm, outputDiv=True)
    p, U, flags, density = simulate.getPUFlagsDensityReference(ob)
    simulate.setConstVals(ob, p, U, flags, density)
    return ob


def gamma53(n):
    return n * U64 / (1.0 - n * U64)


def scales_of_sums(s1, s2, n, threshold):
    """scale_from_sums (tfl_device.cuh) in float32 on the double sums, with and without the contraction
    scale_interval allows."""
    f1, f2 = np.float32(s1), np.float32(s2)
    ss = f1 * f1
    out = []
    for t in (f2 * np.float32(n) + np.float32(-1.0) * ss, np.float32(float(f2) * float(np.float32(n)) - float(ss))):
        t = t / np.float32(float(n) * float(n - 1))
        out.append(max(float(np.sqrt(np.float32(t))), float(np.float32(threshold))))
    return out


def check_sums(sims, U1_ref, threshold, what):
    """Every rank's partial sums against the exact sums of its owned planes, and the rank-order total's scale."""
    total = 0.0
    for q in sims:
        own = U1_ref[:, :, q.dec.z0:q.dec.z1].astype(np.float64).ravel()
        sq = (U1_ref[:, :, q.dec.z0:q.dec.z1] * U1_ref[:, :, q.dec.z0:q.dec.z1]).astype(np.float64).ravel()
        got = q.sums.cpu().numpy()
        for g, x, name in ((got[0], own, "sum"), (got[1], sq, "sum of squares")):
            exact = math.fsum(x)
            bound = gamma53(x.size - 1) * math.fsum(np.abs(x))
            assert abs(g - exact) <= bound, "%s rank %d: %s %.17g, exact %.17g, bound %.3g" % (
                what, q.dec.rank, name, g, exact, bound)
        total = total + q.sums.cpu()
    lo, hi = scale_interval(U1_ref, "std", threshold)
    for sc in scales_of_sums(float(total[0]), float(total[1]), U1_ref.size, threshold):
        assert lo <= sc <= hi, "%s: the total's scale %.9g is outside [%.9g, %.9g]" % (what, sc, lo, hi)


def distances(gnz, bounds):
    """Planes from the nearest rank boundary: 0 for the planes z0 - 1 and z0 either side of one."""
    z = np.arange(gnz)
    return np.min([np.where(z >= b, z - b, b - 1 - z) for b in bounds], axis=0)


def ratio(got, want, E):
    err = np.abs(np.asarray(got, np.float64) - want)
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(err == 0, 0.0, err / E)


def make_model(mnp, mode):
    from fluidnet_b200.model import ProjectionModel
    gm = ProjectionModel.from_model(mnp)
    gm.set_mode(mode)
    return gm


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_slab_steps_per_voxel(case):
    from fluidnet_b200.slab import SlabSimulator
    world, gnz, ny, nx, n, agg, mode, margin = case
    tb, mconf, mnp, bk = problem(case)
    dev = torch.device("cuda", 0)
    sims = [SlabSimulator(tb, mconf, mnp["layers"], dev, rank=r, world=world, margin=margin, banks=bk, conv_mode=mode)
            for r in range(world)]
    assert all(q.model.get_mode() == mode for q in sims)
    gm = make_model(mnp, mode)
    orc = oracle.Oracle()
    dist = distances(gnz, boundaries(case))
    worst = {"p": 0.0, "U": 0.0}
    by_dist = np.zeros(dist.max() + 1)
    for step in range(3):
        what = "%s step %d" % (case_id(case), step)
        state = {k: gather(sims, k).to(dev) for k in sims[0].s}
        pre = pre_projection(state, mconf, gm)
        U1_ref = input_fields(orc, pre["pDiv"].cpu().numpy(), pre["UDiv"].cpu().numpy(),
                              pre["flags"].cpu().numpy())["U1"]
        twins = {}

        def on_sums(sims):
            got = torch.cat([q.dec.owned(q.U1).cpu() for q in sims], dim=2)
            assert same_bits(got, torch.from_numpy(U1_ref)), "%s: U1 differs from the whole grid's" % what
            check_sums(sims, U1_ref, gm.threshold, what)

        def on_project(sims):
            for q in sims:
                twins[q.dec.rank] = check_writes_and_reach(q, n, "%s rank %d" % (what, q.dec.rank))

        lockstep(sims, on_sums, on_project)
        torch.cuda.synchronize()
        for q in sims:
            assert same_bits(q.dec.owned(q.s["pDiv"]), twins[q.dec.rank]), "%s: the step's p is not the twin's" % what
        if step == 0:
            assert same_bits(gather(sims, "density"), pre["density"].cpu()), "%s: density is not bit-exact" % what
        ref = projection_reference(state, mconf, gm, mnp)
        got = {"p": gather(sims, "pDiv").numpy(), "U": gather(sims, "UDiv").numpy()}
        for k in ("p", "U"):
            worst[k] = max(worst[k], check("%s %s" % (what, k), got[k], ref[k], ref["E" + k]))
            per_plane = ratio(got[k], ref[k], ref["E" + k]).max(axis=(0, 1, 3, 4))
            np.maximum.at(by_dist, dist, per_plane)
    assert sims[0].ctx.trace_faults() == 0
    print("slab f64 %s: max err/E p %.3g U %.3g; by distance from a rank boundary: %s" % (
        case_id(case), worst["p"], worst["U"], " ".join("%d:%.3g" % (i, r) for i, r in enumerate(by_dist))))


@pytest.mark.gpu
@pytest.mark.parametrize("n,agg,mode", [(1, None, "tf32x3"), (2, "concat", "tf32"), (3, "add", "tf32x3")])
def test_world1_library_driver_per_voxel(n, agg, mode):
    """NativeSlabSimulator at world 1 (tfl_slab_sim_step, the library's own slab step), two steps, each against the
    float64 projection of its downloaded start state."""
    from fluidnet_b200.slab import NativeSlabSimulator
    case = (1, 32, 16, 16, n, agg, mode, None)
    tb, mconf, mnp, bk = problem(case)
    dev = torch.device("cuda", 0)
    sim = NativeSlabSimulator(tb, mconf, mnp["layers"], dev, rank=0, world=1, banks=bk, conv_mode=mode)
    gm = make_model(mnp, mode)
    const = {k: tb[k] for k in ("flags",) + BC_KEYS}
    try:
        for step in range(2):
            state = {**{k: torch.from_numpy(v) for k, v in sim.download().items()}, **const}
            state = {k: v.to(dev) for k, v in state.items()}
            ref = projection_reference(state, mconf, gm, mnp)
            sim.step()
            torch.cuda.synchronize()
            got = sim.download()
            what = "library slab world 1 N%d %s %s step %d" % (n, agg, mode, step)
            rp = check(what + " p", got["pDiv"], ref["p"], ref["Ep"])
            rU = check(what + " U", got["UDiv"], ref["U"], ref["EU"])
            print("slab f64 %s: max err/E p %.3g U %.3g" % (what, rp, rU))
        sim.check()
    finally:
        sim.close()
