"""Multi-GPU z-slab parity (needs >= 2 GPUs; skipped otherwise): K steps of the convnet step on ONE
domain split across 2 ranks (NCCL halo exchange + 2-double all-reduce) equal the single-GPU run.
Advection / forces are bit-exact; the only reduction whose order changes is the input scale of the
network (sum of two partial sums instead of one), hence 1e-6 * max|field|."""
import pytest
import torch
import torch.multiprocessing as mp

from slab_cases import collect, convnet_problem, free_port, slab_worker

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("native,peer", [(False, False), (True, False), (True, True)],
                         ids=["torch_exchange", "library_nccl", "library_peer_memory"])
@pytest.mark.parametrize("world,n,steps", [(2, 48, 2), (4, 64, 2)])
def test_multi_gpu_slab_matches_single_gpu(world, n, steps, native, peer):
    """native: the whole decomposed step inside libtfl.so (tfl_slab_sim_step, NCCL owned by the context); peer: its
    halos through CUDA-IPC peer memory (push / pull kernels over NVLink) instead of ncclSend / ncclRecv."""
    if torch.cuda.device_count() < world:
        pytest.skip("needs %d GPUs" % world)
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = free_port()
    procs = [ctx.Process(target=slab_worker, args=(r, world, port, n, steps, q, native, peer)) for r in range(world)]
    for p in procs:
        p.start()
    res = collect(procs, q, 150)
    assert len(res) == world and all(r[1] == "ok" for r in res), res


def test_single_rank_slab_driver_matches_fused_step():
    """world == 1 exercises the slab code path (tfl_cnn_stats / _from_sums, set_slab with the whole
    range) on one GPU."""
    from fluidnet_b200 import simulate, model as fmodel
    from fluidnet_b200.slab import SlabSimulator
    batch, mconf, mnp = convnet_problem(32)
    tb = {k: torch.from_numpy(v) for k, v in batch.items()}
    sim = SlabSimulator(tb, mconf, mnp["layers"], torch.device("cuda", 0), rank=0, world=1)
    gb = {k: v.cuda() for k, v in tb.items()}
    gm = fmodel.ProjectionModel(mnp["layers"], True)
    for _ in range(2):
        sim.step()
        simulate.simulate_fused(None, mconf, gb, gm)
    sim.check()
    for k in ("density", "UDiv", "pDiv"):
        want = gb[k].cpu()
        got = sim.gather(k)
        err = (got - want).abs().max().item()
        assert err <= 1e-6 * max(want.abs().max().item(), 1e-6), (k, err)


def test_single_rank_library_slab_step_matches_fused_step():
    """tfl_slab_sim_* with one rank: the C driver of the decomposed step (uploads, slab placement, the split
    projection, downloads) against the fused single-GPU step, no NCCL involved."""
    from fluidnet_b200 import simulate, model as fmodel
    from fluidnet_b200.slab import NativeSlabSimulator
    batch, mconf, mnp = convnet_problem(32)
    tb = {k: torch.from_numpy(v) for k, v in batch.items()}
    sim = NativeSlabSimulator(tb, mconf, mnp["layers"], torch.device("cuda", 0), rank=0, world=1)
    gb = {k: v.cuda() for k, v in tb.items()}
    gm = fmodel.ProjectionModel(mnp["layers"], True)
    for _ in range(2):
        sim.step()
        simulate.simulate_fused(None, mconf, gb, gm)
    sim.check()
    ms, by = sim.exchange_stats()
    assert by == [0, 0, 0] and all(m >= 0 for m in ms)
    for k in ("density", "UDiv", "pDiv"):
        want = gb[k].cpu()
        got = sim.gather(k)
        err = (got - want).abs().max().item()
        assert err <= 1e-6 * max(want.abs().max().item(), 1e-6), (k, err)
    sim.close()


@pytest.mark.parametrize("world,n,steps", [(2, 48, 2), (3, 48, 1)])
def test_emulated_slabs_on_one_gpu(world, n, steps):
    """The complete multi-rank logic (slab geometry, halo widths, split reduction) with every slab on
    one GPU and exchanges served in-process: equals the undivided single-GPU run."""
    from fluidnet_b200 import simulate, model as fmodel
    from fluidnet_b200.slab import SlabSimulator, run_lockstep
    batch, mconf, mnp = convnet_problem(n)
    tb = {k: torch.from_numpy(v) for k, v in batch.items()}
    dev = torch.device("cuda", 0)
    sims = [SlabSimulator(tb, mconf, mnp["layers"], dev, rank=r, world=world) for r in range(world)]
    gb = {k: v.cuda() for k, v in tb.items()}
    gm = fmodel.ProjectionModel(mnp["layers"], True)
    for step in range(steps):
        run_lockstep(sims)
        simulate.simulate(None, mconf, gb, gm)
        for k in ("density", "UDiv", "pDiv"):
            want = gb[k].cpu()
            got = torch.cat([q.dec.owned(q.s[k]).cpu() for q in sims], dim=2)
            err = (got - want).abs()
            scale = max(want.abs().max().item(), 1e-6)
            worst = int(err.reshape(err.shape[0], err.shape[1], err.shape[2], -1).max(3)[0].max(1)[0].argmax())
            assert err.max().item() <= 1e-6 * scale, "step %d %s: %g (scale %g) worst plane z=%d" % (
                step, k, err.max().item(), scale, worst)
            if step == 0 and k == "density":
                assert torch.equal(got, want)            # advection never saw the reduction: bit-exact
    assert sims[0].ctx.trace_faults() == 0
