"""simMethod 'jacobi' on z-slabs: the decomposed step has no reduction, so p, U and density must equal the single-GPU
step bit for bit -- emulated slabs on one GPU (SlabSimulator + run_lockstep), the library driver at one rank and
over 2 / 4 GPUs (skipped on smaller boxes), and the one-launch block kernel against one launch per sweep."""
import ctypes as C

import pytest
import torch
import torch.multiprocessing as mp

from slab_cases import KEYS, jacobi_problem, jacobi_reference

pytestmark = pytest.mark.gpu


# (world, nx, ny, gnz, margin, maxIter or block-relative, forces)
EMU = []
for world in (2, 3, 4):
    for it in (1, "k-1", "k", "k+1", 34, 100):
        EMU.append((world, 32, 24, 6 * world + 1, 2, it, (True, False, True)))
EMU += [
    (2, 32, 24, 16, 3, "k+1", (True, True, False)),            # margin 3, thinnest legal slab
    (2, 32, 24, 17, 3, 34, (False, True, True)),               # uneven slabs
    (3, 32, 24, 20, 2, 34, (False, True, True)),
    (4, 24, 16, 27, 2, 100, (False, False, False)),            # no forces, uneven
    (2, 128, 16, 13, 2, 34, (True, False, True)),              # one-launch block kernel
    (3, 128, 16, 20, 2, 100, (True, True, True)),
    # rank 0 owns 9 planes: the last advection z tile runs past them, and counted faults there (DESIGN.md section 1)
    (3, 128, 16, 26, 3, "k+1", (True, True, False)),
]


def _iters(spec, margin):
    k = 2 * margin + 2
    return {"k-1": k - 1, "k": k, "k+1": k + 1}.get(spec, spec)


@pytest.mark.parametrize("world,nx,ny,gnz,margin,it,forces", EMU)
def test_emulated_slabs_bit_identical(world, nx, ny, gnz, margin, it, forces):
    from fluidnet_b200.slab import SlabSimulator, run_lockstep
    tb, mconf = jacobi_problem(nx, ny, gnz, *forces, max_iter=_iters(it, margin))
    want = jacobi_reference(tb, mconf, 3)
    dev = torch.device("cuda", 0)
    sims = [SlabSimulator(tb, mconf, None, dev, rank=r, world=world, margin=margin) for r in range(world)]
    for step in range(3):
        run_lockstep(sims)
        for k in KEYS:
            got = torch.cat([q.dec.owned(q.s[k]).cpu() for q in sims], dim=2)
            assert torch.equal(got, want[step][k]), "step %d %s: max err %g" % (
                step, k, (got - want[step][k]).abs().max().item())
    assert sims[0].ctx.trace_faults() == 0


@pytest.mark.parametrize("n", [32, 128])
def test_single_rank_library_step_bit_identical(n):
    from fluidnet_b200 import simulate
    from fluidnet_b200.slab import NativeSlabSimulator
    tb, mconf = jacobi_problem(n, n, n, max_iter=34)
    sim = NativeSlabSimulator(tb, mconf, None, torch.device("cuda", 0), rank=0, world=1)
    gb = {k: v.cuda() for k, v in tb.items()}
    for _ in range(2):
        sim.step()
        simulate.simulate_fused(None, mconf, gb)
    sim.check()
    assert sim.jacobi_stats()[0] == 0 and sim.jacobi_stats()[2] == 0
    for k in KEYS:
        assert torch.equal(sim.gather(k), gb[k].cpu()), k
    sim.close()


def test_refusals():
    from fluidnet_b200 import _lib, simulate
    from fluidnet_b200.slab import NativeSlabSimulator, SlabSimulator
    tb, mconf = jacobi_problem(32, 24, 16, max_iter=5)
    dev = torch.device("cuda", 0)
    sim = NativeSlabSimulator(tb, mconf, None, dev, rank=0, world=1)
    lib = sim.ctx.lib
    for method, max_iter, words in [(2, 5, ("'pcg'", "IC(0)")), (0, 5, ("'convnet'", "model")), (1, -1, ("maxIter",))]:
        mc = simulate.make_mconf(mconf)
        mc.sim_method, mc.max_iter = method, max_iter
        assert lib.tfl_slab_sim_step(sim.ctx.h, sim.h, C.byref(mc), None) != 0
        msg = lib.tfl_last_error(sim.ctx.h).decode()
        assert all(w in msg for w in words), msg
    sim.close()
    for bad in (dict(maxIter=0), dict(maxIter=-3), dict(simMethod="pcg")):
        with pytest.raises(ValueError):
            SlabSimulator(tb, dict(mconf, **bad), None, dev, rank=0, world=2)
    assert _lib.load().tfl_slab_jacobi_schedule(16, 2, 0, 2, 0, None, None, 0) == -1


# ---- the block kernel alone --------------------------------------------------------------------------------------
def _block_case(nx, ny, nz, zoff, gnz, seed):
    g = torch.Generator().manual_seed(seed)
    flags = torch.ones(1, 1, nz, ny, nx)                       # fluid
    flags[torch.rand(flags.shape, generator=g) < 0.1] = 2.0    # obstacles
    div = torch.randn(flags.shape, generator=g)
    pa = torch.randn(flags.shape, generator=g)
    pb = torch.randn(flags.shape, generator=g)
    return [t.cuda() for t in (flags, div, pa, pb)]


def _run_block(ctx, flags, div, pa, pb, zoff, gnz, z_lo, z_hi, slo, shi, k, path, is3d=1):
    from fluidnet_b200 import tfluids as t
    a, b = pa.clone(), pb.clone()
    used = C.c_int32(-1)
    if zoff is not None:
        ctx.set_slab(zoff, gnz, z_lo, z_hi)
    try:
        rc = ctx.lib.tfl_jacobi_slab_block(ctx.h, t._grid(a), t._grid(b), t._grid(flags), t._grid(div), is3d, z_lo, z_hi,
                                           slo, shi, k, path, C.byref(used))
    finally:
        if zoff is not None:
            ctx.clear_slab()
    torch.cuda.synchronize()
    return rc, a, b, used.value


@pytest.mark.parametrize("k", [1, 2, 3, 5, 6, 8])
@pytest.mark.parametrize("shape", ["interior", "bottom_end", "top_end"])
def test_block_kernel_equals_per_sweep_launches(k, shape):
    """Interior slab (both sides shrink), and the first / last rank (one side runs to the global end)."""
    from fluidnet_b200 import tfluids
    ctx = tfluids.context()
    nx, ny, nz, halo = 128, 16, 40, 8
    zoff, gnz, z_lo, z_hi, slo, shi = {"interior": (50, 200, halo + 1 - k, nz - halo - 1 + k, 1, 1),
                                       "bottom_end": (0, 200, 0, nz - halo - 1 + k, 0, 1),
                                       "top_end": (160, 200, halo + 1 - k, nz, 1, 0)}[shape]
    flags, div, pa, pb = _block_case(nx, ny, nz, zoff, gnz, seed=k)
    rc0, a0, b0, u0 = _run_block(ctx, flags, div, pa, pb, zoff, gnz, z_lo, z_hi, slo, shi, k, 0)
    rc1, a1, b1, u1 = _run_block(ctx, flags, div, pa, pb, zoff, gnz, z_lo, z_hi, slo, shi, k, 1)
    assert rc0 == 0 and rc1 == 0 and (u0, u1) == (0, 1), ctx.lib.tfl_last_error(ctx.h)
    assert torch.equal(a0, a1) and torch.equal(b0, b1)
    out = b1 if k & 1 else a1
    untouched = torch.ones(nz, dtype=torch.bool)
    untouched[z_lo:z_hi] = False
    assert torch.equal(a1[:, :, untouched], pa[:, :, untouched]) and torch.equal(b1[:, :, untouched], pb[:, :, untouched])
    assert not torch.equal(out, pa if k & 1 == 0 else pb)


def test_block_kernel_dispatch_branches():
    from fluidnet_b200 import tfluids
    ctx = tfluids.context()
    # nx % 128 != 0: the one-launch path is refused, the automatic one falls back to per-sweep launches
    flags, div, pa, pb = _block_case(96, 16, 24, 10, 100, seed=1)
    rc, *_ = _run_block(ctx, flags, div, pa, pb, 10, 100, 4, 20, 1, 1, 4, 1)
    assert rc != 0
    rc, a, b, used = _run_block(ctx, flags, div, pa, pb, 10, 100, 4, 20, 1, 1, 4, -1)
    assert rc == 0 and used == 0
    # a range too large to be co-resident (4.2M cells): per-sweep launches
    flags, div, pa, pb = _block_case(256, 256, 66, 10, 300, seed=2)
    rc, *_ = _run_block(ctx, flags, div, pa, pb, 10, 300, 1, 65, 1, 1, 2, 1)
    assert rc != 0
    rc, a, b, used = _run_block(ctx, flags, div, pa, pb, 10, 300, 1, 65, 1, 1, 2, -1)
    assert rc == 0 and used == 0
    # 2.6M cells: only the 6-plane blocks fit; same bits as per-sweep launches
    flags, div, pa, pb = _block_case(256, 256, 42, 10, 300, seed=3)
    r0 = _run_block(ctx, flags, div, pa, pb, 10, 300, 1, 41, 1, 1, 5, 0)
    r1 = _run_block(ctx, flags, div, pa, pb, 10, 300, 1, 41, 1, 1, 5, 1)
    assert r0[0] == 0 and r1[0] == 0 and r1[3] == 1
    assert torch.equal(r0[1], r1[1]) and torch.equal(r0[2], r1[2])
    # reads past the local storage are refused
    rc, *_ = _run_block(ctx, flags, div, pa, pb, 10, 300, 0, 41, 1, 1, 2, -1)
    assert rc != 0


@pytest.mark.parametrize("nz,ny,nx,is3d,iters", [(24, 16, 128, 1, 34), (1, 40, 36, 0, 20), (1, 64, 128, 0, 7)])
def test_block_equals_jacobi_operator(nz, ny, nx, is3d, iters):
    """On a whole grid (no slab placement) one block of `iters` sweeps from p = 0 is the Jacobi solve; 2-D grids take
    the per-sweep path."""
    from fluidnet_b200 import tfluids, synth
    ctx = tfluids.context()
    flags = torch.from_numpy(synth.make_flags(nx, ny, nz if is3d else 1, bool(is3d), nb=1, geometry=True)).cuda()
    div = torch.randn(flags.shape, generator=torch.Generator().manual_seed(5)).cuda()
    zero = torch.zeros_like(div)
    rc, a, b, used = _run_block(ctx, flags, div, zero, zero, None, None, 0, flags.shape[2], 0, 0, iters, -1, is3d)
    assert rc == 0, ctx.lib.tfl_last_error(ctx.h)
    assert used == (1 if is3d else 0)
    p = torch.empty_like(div)
    tfluids.solveLinearSystemJacobi(p, flags, div, bool(is3d), 0, iters)
    assert torch.equal(b if iters & 1 else a, p)


# ---- several GPUs --------------------------------------------------------------------------------------------------
def _worker(rank, world, port, q, peer):
    import os
    import torch.distributed as dist
    try:
        os.environ["MASTER_ADDR"] = "127.0.0.1"
        os.environ["MASTER_PORT"] = str(port)
        torch.cuda.set_device(rank)
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
        from fluidnet_b200.slab import NativeSlabSimulator
        tb, mconf = jacobi_problem(128, 32, 64, max_iter=34)
        sim = NativeSlabSimulator(tb, mconf, None, torch.device("cuda", rank), rank, world, peer_halos=peer)
        for _ in range(2):
            sim.step()
        sim.check()
        n, ms, by = sim.jacobi_stats()
        assert n == 5 and by > 0, (n, ms, by)
        got = {k: sim.gather(k) for k in KEYS}
        if rank == 0:
            want = jacobi_reference(tb, mconf, 2)[-1]
            for k in KEYS:
                assert torch.equal(got[k], want[k]), k
        dist.barrier()
        sim.close()
        dist.destroy_process_group()
        q.put((rank, "ok"))
    except Exception:       # pragma: no cover
        import traceback
        q.put((rank, "FAIL: %s" % traceback.format_exc()))
        raise


@pytest.mark.parametrize("peer", [False, True], ids=["nccl", "peer_memory"])
@pytest.mark.parametrize("world", [2, 4])
def test_multi_gpu_library_step_bit_identical(world, peer):
    if torch.cuda.device_count() < world:
        pytest.skip("needs %d GPUs" % world)
    from slab_cases import collect, free_port
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q, peer)) for r in range(world)]
    for p in procs:
        p.start()
    res = collect(procs, q, 150)
    assert len(res) == world and all(r[1] == "ok" for r in res), res
