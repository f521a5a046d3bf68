"""Banked projection networks on z-slabs: the 3-D 'default' graph with banks split at stage 1 and joined at stage 3,
on the tensor cores (3xTF32, TF32).  Each rank pools the global grid's 2x2x2 blocks whatever its plane offset, runs
every bank's layers on the coarse planes the join needs and joins with the bank's z phase; the slab margin is at
least tfl_slab_cnn_margin(banksNum) (tests/test_slab_cnn_reach.py derives it).

Against the single-GPU step with the same model: the advected density of the first step bit for bit, p and U within
1e-6 of each field's max in 3xTF32 (the input scale's sum is split over the ranks, as in tests/test_gpu_slab.py) and
3e-3 in TF32 (a last-bit change of the scale can flip a TF32 input rounding).  Kernel level: the pyramid with a z
phase and the join with bank offsets on a restricted plane range, against float64 with the bound of
tests/test_gpu_conv_tc_join.py, planes outside the range untouched and NaN in every bank plane the range does not
need.  Refusals name the z-slab and launch nothing."""
import ctypes as C
import zlib

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from scenes import banks
from slab_cases import BANKED_TOL, banked_problem, refused, single_gpu
from tc_conv import KAPPA, SENTINEL, is_sentinel, join_reference, layout, pack

pytestmark = pytest.mark.gpu


def _close(got, want, tol, what):
    err = (got - want).abs().max().item()
    scale = max(want.abs().max().item(), 1e-6)
    assert err <= tol * scale, "%s: %g (scale %g)" % (what, err, scale)


# (world, gnz, ny, nx, banksNum, aggregate, mode, margin or None): rank boundaries at odd planes (40 over 3: 14, 27)
# and at 3 / 2 mod 4 (44 over 3: 15, 30), uneven slabs, the thinnest legal slab (halo 8: 32 over 4; halo 14: 28 over
# 2), a margin above the minimum.
EMU = [
    (2, 32, 16, 16, 2, "concat", "tf32x3", None),
    (3, 40, 16, 16, 2, "add", "tf32x3", None),
    (3, 40, 16, 24, 2, "concat", "tf32", None),
    (4, 32, 16, 16, 2, "concat", "tf32x3", 3),
    (3, 44, 16, 16, 3, "concat", "tf32x3", None),
    (3, 44, 16, 16, 3, "add", "tf32", None),
    (2, 28, 16, 16, 3, "add", "tf32x3", 6),
    (4, 64, 16, 16, 3, "concat", "tf32x3", 7),
]


def emu_id(c):
    return "w%d-%dx%dx%d-N%d-%s-%s-m%s" % c


@pytest.mark.parametrize("case", EMU, ids=emu_id)
def test_emulated_slabs_match_single_gpu(case):
    from fluidnet_b200.slab import SlabSimulator, run_lockstep, cnn_margin
    world, gnz, ny, nx, n, agg, mode, margin = case
    bk = banks(n, agg)
    tb, mconf, mnp = banked_problem(gnz, ny, nx, bk)
    dev = torch.device("cuda", 0)
    sims = [SlabSimulator(tb, mconf, mnp["layers"], dev, rank=r, world=world, margin=margin, banks=bk, conv_mode=mode)
            for r in range(world)]
    assert all(q.margin == (margin or cnn_margin(n)) for q in sims)
    gb, step = single_gpu(tb, mconf, mnp, bk, mode)
    for it in range(3 if world < 4 else 2):
        run_lockstep(sims)
        step()
        for k in ("density", "UDiv", "pDiv"):
            got = torch.cat([q.dec.owned(q.s[k]).cpu() for q in sims], dim=2)
            want = gb[k].cpu()
            if it == 0 and k == "density":
                assert torch.equal(got, want), "density is not bit-exact"
            _close(got, want, BANKED_TOL[mode], "step %d %s" % (it, k))
    assert sims[0].ctx.trace_faults() == 0


@pytest.mark.parametrize("native", [False, True], ids=["python", "library"])
@pytest.mark.parametrize("n,agg", [(2, "concat"), (3, "add")])
def test_single_rank_drivers_match_fused_step(native, n, agg):
    from fluidnet_b200.slab import SlabSimulator, NativeSlabSimulator
    bk = banks(n, agg)
    tb, mconf, mnp = banked_problem(32, 32, 32, bk)
    cls = NativeSlabSimulator if native else SlabSimulator
    sim = cls(tb, mconf, mnp["layers"], torch.device("cuda", 0), rank=0, world=1, banks=bk)
    gb, step = single_gpu(tb, mconf, mnp, bk, "tf32x3", fused=True)
    for _ in range(2):
        sim.step()
        step()
    sim.check()
    if native:
        ms, by = sim.exchange_stats()
        assert by == [0, 0, 0] and all(m >= 0 for m in ms)
    for k in ("density", "UDiv", "pDiv"):
        _close(sim.gather(k), gb[k].cpu(), 1e-6, k)
    if native:
        sim.close()


def _hooks():
    from fluidnet_b200 import _lib
    lib = _lib.load()
    P = C.c_void_p
    lib.tfl_debug_tc_pyramid.argtypes = [P, P, P] + [C.c_int] * 8
    lib.tfl_debug_conv3_tc_join_slab.argtypes = ([P, C.POINTER(P), C.c_int, C.c_int, P, P, P, P] + [C.c_int] * 6
                                                 + [C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.c_int, C.c_int])
    return lib


@pytest.mark.parametrize("phase", [0, 1])
def test_pyramid_with_z_phase_on_a_plane_range(phase):
    """Output planes [z_lo, z_hi) pool input planes 2 z + phase, 2 z + phase + 1 in k_pool's order (bit for bit);
    the other output planes keep their bits and the input planes outside the pooled ones hold NaN."""
    from fluidnet_b200 import tfluids
    nb, nz_in, ny, nx = 2, 13, 6, 10
    nz_out, z_lo, z_hi = 6, 1, 5
    rs = np.random.RandomState(7 + phase)
    x = rs.uniform(-1, 1, (nb, 3, nz_in, ny, nx)).astype(np.float32)
    px, py = layout(nb, nz_in, ny, nx)
    hin = pack(x, px, py, fill_unused=np.nan)
    used = np.zeros(nz_in, bool)
    used[2 * z_lo + phase:2 * z_hi + phase] = True
    hin[:, :, 1:nz_in + 1][:, :, ~used] = np.nan
    qx, qy = layout(nb, nz_out, ny // 2, nx // 2)
    hout = np.full((nb, 2, nz_out + 2, qy, qx, 4), SENTINEL, np.float32)
    din, dout = torch.from_numpy(hin).cuda(), torch.from_numpy(hout).cuda()
    ctx = tfluids._ctx_for(din)
    ctx.check(_hooks().tfl_debug_tc_pyramid(ctx.h, din.data_ptr(), dout.data_ptr(), nb, nz_in, ny, nx, nz_out, phase,
                                            z_lo, z_hi))
    got = dout.cpu().numpy()
    want = hout.copy()
    for z in range(z_lo, z_hi):
        acc = np.zeros((nb, ny // 2, nx // 2, 3), np.float32)
        for dz in range(2):
            for dy in range(2):
                for dx in range(2):
                    v = x[:, :, 2 * z + phase + dz, dy::2, dx::2].transpose(0, 2, 3, 1)
                    acc = (acc + v).astype(np.float32)
        want[:, 0, z + 1, 1:ny // 2 + 1, 1:nx // 2 + 1, :3] = acc / np.float32(8.0)
        want[:, 0, z + 1, 1:ny // 2 + 1, 1:nx // 2 + 1, 3] = 0.0
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


# (global nz, ny, nx, banksNum, zoff, local nz, z_lo, z_hi): odd and even offsets, banks starting at a rounded-up
# coarse plane, a range reaching the last plane with a full stencil.
JOIN = [(32, 16, 16, 3, 5, 20, 4, 15), (32, 8, 40, 2, 7, 14, 2, 11), (48, 16, 16, 3, 10, 22, 3, 21),
        (24, 8, 8, 2, 0, 24, 3, 9)]


@pytest.mark.parametrize("case", JOIN, ids=lambda c: "g%d-%dx%d-N%d-zoff%d-nz%d-%d:%d" % c)
@pytest.mark.parametrize("agg", ["concat", "add"])
@pytest.mark.parametrize("split", [1, 0], ids=["tf32x3", "tf32"])
def test_join_with_bank_offsets_on_a_plane_range(split, agg, case):
    """The join of a slab's banks (bank i from global coarse plane ceil(zoff / 2^i)) on local planes [z_lo, z_hi)
    equals the whole grid's float64 join at global planes zoff + z, within the kappa S bound."""
    from fluidnet_b200 import tfluids
    gnz, ny, nx, n, zoff, nz, z_lo, z_hi = case
    what = "join-slab %s %s %s" % (split, agg, case)
    rs = np.random.RandomState(zlib.crc32(what.encode()))
    full = [rs.uniform(0.0, 1.0, (1, 8, gnz >> i, ny >> i, nx >> i)).astype(np.float32) for i in range(n)]
    cin = 8 * n if agg == "concat" else 8
    bw, bt = 1.0 / np.sqrt(cin * 27), 1.0 / np.sqrt(8)
    w = rs.uniform(-bw, bw, (8, cin, 3, 3, 3)).astype(np.float32)
    b = rs.uniform(-bw, bw, 8).astype(np.float32)
    tail = rs.uniform(-bt, bt, 81).astype(np.float32)
    org = [zoff] + [-(-zoff // 2 ** i) for i in range(1, n)]
    bnz = [nz] + [((zoff + nz) >> i) - org[i] for i in range(1, n)]
    dev = []
    for i in range(n):
        x = full[i][:, :, org[i]:org[i] + bnz[i]]
        px, py = layout(1, bnz[i], ny >> i, nx >> i)
        buf = pack(x, px, py)
        buf[:, :, :, :, (nx >> i) + 2:, :] = np.nan
        lo, hi = ((zoff + z_lo - 1) >> i) - org[i], ((zoff + z_hi) >> i) - org[i]      # planes the range reads
        keep = np.zeros(bnz[i], bool)
        keep[max(lo, 0):hi + 1] = True
        buf[:, :, 1:bnz[i] + 1][:, :, ~keep] = np.nan
        dev.append(torch.from_numpy(buf).cuda())
    p = torch.full((1, nz, ny, nx), float(SENTINEL), device="cuda")
    ctx = tfluids._ctx_for(p)
    ptrs = (C.c_void_p * n)(*[d.data_ptr() for d in dev])
    ctx.check(_hooks().tfl_debug_conv3_tc_join_slab(ctx.h, ptrs, n, 1 if agg == "add" else 0, p.data_ptr(),
                                                     w.ctypes.data, b.ctypes.data, tail.ctypes.data, split, 1, nz, ny,
                                                     nx, zoff, (C.c_int32 * n)(*bnz), (C.c_int32 * n)(*org), z_lo, z_hi))
    got = p.cpu().numpy()
    outside = np.ones(nz, bool)
    outside[z_lo:z_hi] = False
    assert is_sentinel(got[:, outside]).all(), "%s: a plane outside the range was written" % what
    got = got[:, z_lo:z_hi]
    assert np.isfinite(got).all(), "%s: a NaN plane was read" % what
    ref, bound = join_reference(full, agg, w, b, tail, KAPPA[split])
    ref, bound = ref[:, zoff + z_lo:zoff + z_hi], bound[:, zoff + z_lo:zoff + z_hi]
    err = np.abs(got.astype(np.float64) - ref)
    assert (err <= bound).all(), "%s: %d voxels over the bound (worst ratio %.2f)" % (
        what, (err > bound).sum(), (err / np.maximum(bound, 1e-300)).max())


def test_refusals_name_the_z_slab():
    from fluidnet_b200 import simulate, synth, tfluids, model as fmodel
    from fluidnet_b200.slab import SlabSimulator, NativeSlabSimulator
    dev = torch.device("cuda", 0)
    b2 = banks(2, "concat")
    tb, mconf, mnp2 = banked_problem(32, 16, 16, b2)
    # a margin one below the minimum, from both drivers
    for cls in (SlabSimulator, NativeSlabSimulator):
        with pytest.raises(ValueError, match="margin >= 3"):
            cls(tb, mconf, mnp2["layers"], dev, rank=0, world=2, margin=2, banks=b2)
    # the C step: a single-bank slab at margin 2 (and a global grid of 30 planes) stepped with other models
    single = synth.make_model(True)
    sim = NativeSlabSimulator(tb, mconf, single["layers"], dev, rank=0, world=1)
    tb30, _, _ = banked_problem(30, 16, 16, b2)
    sim30 = NativeSlabSimulator(tb30, mconf, single["layers"], dev, rank=0, world=1, margin=6)
    ctx, mc = sim.ctx, simulate.make_mconf(mconf)
    step = lambda s, m: lambda: ctx.lib.tfl_slab_sim_step(ctx.h, s.h, C.byref(mc), m.h)
    m2 = fmodel.ProjectionModel(mnp2["layers"], True, banks=b2)
    assert b"margin >= 3" in refused(ctx, step(sim, m2))
    m3 = fmodel.ProjectionModel(synth.make_model(True, banks=banks(3, "add"))["layers"], True, banks=banks(3, "add"))
    assert b"divisible" in refused(ctx, step(sim30, m3))
    other = banks(2, "concat", s=2, j=4)
    m24 = fmodel.ProjectionModel(synth.make_model(True, banks=other)["layers"], True, banks=other)
    assert b"tensor-core path only" in refused(ctx, step(sim, m24))
    m2.set_mode("fp32")
    assert b"tensor-core path only" in refused(ctx, step(sim, m2))
    tog = synth.make_model(True, model_type="tog")
    mt = fmodel.ProjectionModel(tog["layers"], True, pool=tog.get("pool"), up=tog.get("up"))
    assert b"tensor-core path only" in refused(ctx, step(sim, mt))
    # tfl_cnn_project_from_sums under a slab placement whose margin is too small
    m2.set_mode("tf32x3")
    g = torch.zeros(1, 1, 16, 16, 16, device=dev)
    u = torch.zeros(1, 3, 16, 16, 16, device=dev)
    sums = torch.zeros(2, dtype=torch.float64, device=dev)
    ctx.set_slab(8, 32, 7, 9)
    try:
        ctx.check(ctx.lib.tfl_set_slab_margin(ctx.h, 2))
        msg = refused(ctx, lambda: ctx.lib.tfl_cnn_project_from_sums(
            ctx.h, m2.h, tfluids._grid(g), tfluids._grid(u), tfluids._grid(g), C.c_void_p(sums.data_ptr()),
            tfluids._grid(g), tfluids._grid(u), C.c_float(1e-5)))
        assert b"margin >= 3" in msg
        ctx.check(ctx.lib.tfl_set_slab_margin(ctx.h, 3))      # margin fine, 7 ghost planes below: too shallow
        msg = refused(ctx, lambda: ctx.lib.tfl_cnn_project_from_sums(
            ctx.h, m2.h, tfluids._grid(g), tfluids._grid(u), tfluids._grid(g), C.c_void_p(sums.data_ptr()),
            tfluids._grid(g), tfluids._grid(u), C.c_float(1e-5)))
        assert b"ghost planes" in msg
    finally:
        ctx.clear_slab()
        ctx.lib.tfl_set_slab_margin(ctx.h, 2)
    sim.close()
    sim30.close()


def _worker(rank, world, port, gnz, steps, q, native, peer):
    import os
    import torch.distributed as dist
    try:
        os.environ["MASTER_ADDR"] = "127.0.0.1"
        os.environ["MASTER_PORT"] = str(port)
        torch.cuda.set_device(rank)
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
        from fluidnet_b200.slab import SlabSimulator, NativeSlabSimulator
        bk = banks(2, "concat")
        tb, mconf, mnp = banked_problem(gnz, 16, 16, bk)
        kw = {"peer_halos": peer} if native else {}
        sim = (NativeSlabSimulator if native else SlabSimulator)(tb, mconf, mnp["layers"], torch.device("cuda", rank),
                                                               rank, world, banks=bk, **kw)
        if native and peer:
            assert sim.halo_transport.startswith("peer memory"), sim.halo_transport
        for _ in range(steps):
            sim.step()
        sim.check()
        got = {k: sim.gather(k) for k in ("density", "UDiv", "pDiv")}
        if rank == 0:
            gb, step = single_gpu(tb, mconf, mnp, bk, "tf32x3")
            for _ in range(steps):
                step()
            for k in ("density", "UDiv", "pDiv"):
                _close(got[k], gb[k].cpu(), 1e-6, k)
        dist.barrier()
        dist.destroy_process_group()
        q.put((rank, "ok"))
    except Exception:       # pragma: no cover
        import traceback
        q.put((rank, "FAIL: %s" % traceback.format_exc()))
        raise


@pytest.mark.parametrize("native,peer", [(False, False), (True, False), (True, True)],
                         ids=["torch_exchange", "library_nccl", "library_peer_memory"])
@pytest.mark.parametrize("world,gnz", [(2, 32), (4, 44)])
def test_multi_gpu_banked_slabs_match_single_gpu(world, gnz, native, peer):
    from slab_cases import collect, free_port
    if torch.cuda.device_count() < world:
        pytest.skip("needs %d GPUs" % world)
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, gnz, 2, q, native, peer)) for r in range(world)]
    for p in procs:
        p.start()
    res = collect(procs, q, 150)
    assert len(res) == world and all(r[1] == "ok" for r in res), res
