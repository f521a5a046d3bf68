"""tfl_launch_count against the kernels that really ran: each case runs once to warm up, then under torch.profiler
with CUDA activities, and the number of kernel events (memcpy and memset left out) must equal what the call added to
the context's tally.  The cases walk the projection network's drivers: tfl_cnn_project on the fp32 path (plain loop
and graph executor) and on the tensor cores (single bank, banked 'mres' and 'dilate' stacks, batch statistics, the
pressure skip), the fused tfl_simulate_step, and a single-rank tfl_slab_sim_step with a banked model."""
import pytest
import torch

from fluidnet_b200.model import ProjectionModel
from scenes import banks, fields_with_random_p, plume_batch, step_mconf
from step_cases import tally_and_kernels

pytestmark = pytest.mark.gpu


def _check(ctx, call, what):
    tally, kernels = tally_and_kernels(ctx, call)
    assert tally == sum(kernels.values()), (what, "tallied %d, ran %d" % (tally, sum(kernels.values())), dict(kernels))


# (id, synth.make_model keywords, mode, grid nz ny nx)
PROJECT = [
    ("default-fp32", {}, "fp32", (16, 16, 16)),
    ("default-tf32", {}, "tf32", (16, 16, 16)),
    ("default-tf32x3", {}, "tf32x3", (16, 16, 16)),
    ("mres3-concat-tf32x3", {"banks": banks(3, "concat", "mres")}, "tf32x3", (16, 16, 16)),
    ("mres3-concat-fp32", {"banks": banks(3, "concat", "mres")}, "fp32", (16, 16, 16)),
    ("mres3-add-tf32x3", {"banks": banks(3, "add", "mres")}, "tf32x3", (16, 16, 16)),
    ("mres3-add-fp32", {"banks": banks(3, "add", "mres")}, "fp32", (16, 16, 16)),
    # 2 does not divide 15: the short phases of the dilated bank are re-zeroed
    ("dilate2-concat-tf32x3", {"banks": banks(2, "concat", "dilate")}, "tf32x3", (15, 16, 15)),
    ("dilate2-add-fp32", {"banks": banks(2, "add", "dilate")}, "fp32", (15, 16, 15)),
    ("bn-batch-tf32x3", {"batch_norm": {"train": True}}, "tf32x3", (16, 16, 16)),
    ("bn-batch-fp32", {"batch_norm": {"train": True}}, "fp32", (16, 16, 16)),
    ("skip-tf32x3", {"inputs": {"addPressureSkip": True}}, "tf32x3", (16, 16, 16)),
    ("skip-div-scale-fp32", {"inputs": {"addPressureSkip": True, "normalizeInputChan": "div"}}, "fp32", (16, 16, 16)),
    ("tog-fp32", {"model_type": "tog"}, "fp32", (16, 16, 16)),
]


@pytest.mark.parametrize("case", PROJECT, ids=[c[0] for c in PROJECT])
def test_cnn_project_tallies_the_kernels_it_runs(case):
    from fluidnet_b200 import synth
    name, kw, mode, (nz, ny, nx) = case
    gm = ProjectionModel.from_model(synth.make_model(True, **kw))
    gm.set_mode(mode)
    f = {k: torch.from_numpy(v).cuda() for k, v in fields_with_random_p(nz, ny, nx).items()}
    out = (torch.empty_like(f["pDiv"]), torch.empty_like(f["UDiv"]))
    _check(gm.ctx, lambda: gm.forward((f["pDiv"], f["UDiv"], f["flags"]), out=out), name)


def _step_problem(n, bk):
    from fluidnet_b200 import synth
    return plume_batch(n, inflow=n / 128.0 * 4), step_mconf(n), synth.make_model(True, banks=bk)


@pytest.mark.parametrize("bk", [None, banks(2, "concat", "mres")], ids=["default", "mres2-concat"])
def test_fused_step_tallies_the_kernels_it_runs(bk):
    from fluidnet_b200 import simulate
    batch, mconf, mnp = _step_problem(32, bk)
    gm = ProjectionModel.from_model(mnp)
    gm.set_mode("tf32x3")
    gb = {k: torch.from_numpy(v).cuda() for k, v in batch.items()}
    _check(gm.ctx, lambda: simulate.simulate_fused(None, mconf, gb, gm), "tfl_simulate_step")


def test_single_rank_slab_step_tallies_the_kernels_it_runs():
    from fluidnet_b200.slab import NativeSlabSimulator
    bk = banks(2, "concat")
    batch, mconf, mnp = _step_problem(32, bk)
    tb = {k: torch.from_numpy(v) for k, v in batch.items()}
    sim = NativeSlabSimulator(tb, mconf, mnp["layers"], torch.device("cuda", 0), rank=0, world=1, banks=bk)
    try:
        _check(sim.ctx, sim.step, "tfl_slab_sim_step")
    finally:
        sim.close()
