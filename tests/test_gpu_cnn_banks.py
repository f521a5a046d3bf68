"""Multi-resolution banks of the projection network (lib/model.lua:252-361) on the GPU: model:forward against the
CPU restatement (tests/bank_oracle.py, pinned on torch.nn.functional by tests/test_oracle_model_banks.py), the
whole step, CUDA-graph replay, model reuse across grids, and the argument errors.

The 3-D 'default' graph with banks split at stage 1 and joined at stage 3 also runs on the tensor cores (3xTF32 by
default, TF32); every other banked graph runs on the fp32 path.  Per batch entry: scale within 1e-5 relative, p and
U within 2e-5 of the entry's max (fp32, 3xTF32) or 3e-3 (TF32), and the zero pattern of U exact (the class of
tests/test_gpu_step.py)."""
import ctypes as C

import numpy as np
import pytest
import torch

import oracle
from bank_oracle import model_forward_banked
from fluidnet_b200 import synth
from fluidnet_b200 import model as fmodel
from fluidnet_b200._lib import TflError

pytestmark = pytest.mark.gpu


def banks(num, agg, s=1, j=3):
    return {"num": num, "split_stage": s, "join_stage": j, "aggregate": agg}


def make_gpu(mnp, threshold=1e-5):
    return fmodel.ProjectionModel(mnp["layers"], mnp["is3D"], normalizeInputThreshold=threshold, pool=mnp.get("pool"),
                                  up=mnp.get("up"), poolType=mnp.get("poolType", "avg"),
                                  nonlinType=mnp.get("nonlinType", "relu"), banks=mnp.get("banks"))


def make_batch(shape, is3d, nb=1, seed=1234, plume=False):
    nz, ny, nx = shape
    flags = synth.make_flags(nx, ny, nz, is3d, nb=nb, geometry=True)
    U = synth.make_smooth_velocity(flags, is3d, amp=3.0, seed=seed)
    oracle.Oracle().setWallBcsForward(U, flags)
    batch = {"pDiv": np.zeros_like(flags), "UDiv": U, "flags": flags, "density": synth.make_density(flags)}
    if plume:
        oracle.create_plume_bcs(batch, [1.0], nx / 128.0 * 4, 0.15)
    return batch


def close(got, want, tol, what):
    err = np.abs(got.astype(np.float64) - want.astype(np.float64)).max()
    scale = max(np.abs(want).max(), 1e-6)
    assert err <= tol * scale, "%s: max err %g vs scale %g" % (what, err, scale)


def inputs_of(batch, seed=77):
    p0 = (synth.make_density(batch["flags"], seed=seed) - np.float32(0.5)) * np.float32(0.1)
    return p0, tuple(torch.from_numpy(a).cuda() for a in (p0, batch["UDiv"], batch["flags"]))


# (is3d, model_type, banks, (nz, ny, nx), nb).  3-D coarse banks of nx 29, 30, 31 (tile edges of the
# tensor-core layout, should banks move there), ny not a multiple of 4 or 8, a coarse grid with a 1-voxel
# dimension; 2-D 'default' and 'tog' with banks; a non-default split / join.
FORWARD = {
    "3d-n2-concat-x29": (True, "default", banks(2, "concat"), (6, 10, 58), 2),
    "3d-n2-add-x30": (True, "default", banks(2, "add"), (4, 14, 60), 2),
    "3d-n3-concat-x31": (True, "default", banks(3, "concat"), (8, 20, 124), 2),
    "3d-n3-add-z1": (True, "default", banks(3, "add"), (4, 12, 24), 2),
    "3d-n2-concat-s2j4": (True, "default", banks(2, "concat", 2, 4), (6, 10, 12), 2),
    "3d-yang-n2-add": (True, "yang", banks(2, "add", 1, 2), (6, 8, 10), 1),
    "2d-n2-concat": (False, "default", banks(2, "concat"), (1, 36, 52), 2),
    "2d-n3-add": (False, "default", banks(3, "add"), (1, 40, 36), 1),
    "2d-tog-n2-concat": (False, "tog", banks(2, "concat"), (1, 32, 48), 2),
    "3d-tog-n2-add": (True, "tog", banks(2, "add"), (16, 16, 24), 1),
}


MODE_TOL = {"fp32": 2e-5, "tf32x3": 2e-5, "tf32": 3e-3}


def tc_covered(is3d, model_type, bk):
    return is3d and model_type == "default" and bk["split_stage"] == 1 and bk["join_stage"] == 3


@pytest.mark.parametrize("mode", ["default", "fp32", "tf32"])
@pytest.mark.parametrize("case", list(FORWARD))
def test_banked_forward(case, mode):
    orc = oracle.Oracle()
    is3d, model_type, bk, shape, nb = FORWARD[case]
    covered = tc_covered(is3d, model_type, bk)
    if mode != "default" and not covered:
        pytest.skip("fp32 only: the default mode is the only mode")
    batch = make_batch(shape, is3d, nb=nb)
    mnp = synth.make_model(is3d, model_type=model_type, banks=bk)
    p0, inp = inputs_of(batch)
    wp, wU, wscale = model_forward_banked(orc, mnp, p0, batch["UDiv"], batch["flags"])
    gm = make_gpu(mnp)
    assert gm.get_mode() == ("tf32x3" if covered else "fp32")
    if mode != "default":
        gm.set_mode(mode)
    tol = MODE_TOL[gm.get_mode()]
    gp, gU = gm.forward(inp, return_scale=True)
    gp, gU = gp.cpu().numpy(), gU.cpu().numpy()
    for b in range(nb):
        assert abs(gm.last_scale[b] - wscale[b]) <= 1e-5 * wscale[b], (b, gm.last_scale, wscale)
        close(gp[b], wp[b], tol, "p[%d]" % b)
        close(gU[b], wU[b], tol, "U[%d]" % b)
    assert np.array_equal(gU == 0, wU == 0)


@pytest.mark.parametrize("is3d", [True, False], ids=["3d", "2d"])
def test_one_bank_is_the_single_bank_graph(is3d):
    """tfl_cnn_create_banked with num = 1 builds exactly the tfl_cnn_create_graph model: same bits, same default mode."""
    shape = (8, 12, 16) if is3d else (1, 24, 20)
    batch = make_batch(shape, is3d, nb=2)
    plain = synth.make_model(is3d)
    one = dict(plain, banks=banks(1, "concat"))
    _, inp = inputs_of(batch)
    a, b = make_gpu(plain), make_gpu(one)
    assert a.get_mode() == b.get_mode()
    for x, y in zip(a.forward(inp), b.forward(inp)):
        assert torch.equal(x.view(torch.int32), y.view(torch.int32))


@pytest.mark.parametrize("agg", ["concat", "add"])
def test_banked_model_across_shapes_and_modes(agg):
    """One banked model through grid, batch and mode changes equals a fresh model each time: the per-bank padded
    buffers are reallocated with the grid and their zero borders survive between calls."""
    mnp = synth.make_model(True, banks=banks(3, agg))
    gm = make_gpu(mnp)
    for shape, nb, mode, seed in (((8, 12, 16), 1, "tf32x3", 0), ((12, 8, 20), 2, "tf32", 1),
                                  ((8, 12, 16), 1, "fp32", 2), ((8, 12, 16), 1, "tf32x3", 3), ((4, 4, 8), 3, "tf32x3", 4),
                                  ((12, 8, 20), 2, "tf32x3", 5)):
        batch = make_batch(shape, True, nb=nb, seed=1234 + seed)
        _, inp = inputs_of(batch, seed=77 + seed)
        gm.set_mode(mode)
        fresh = make_gpu(mnp)
        fresh.set_mode(mode)
        for got, want, k in zip(gm.forward(inp), fresh.forward(inp), ("p", "U")):
            close(got.cpu().numpy(), want.cpu().numpy(), 1e-6, "%s nb%d %s %s" % (shape, nb, mode, k))


@pytest.mark.parametrize("bk", [banks(2, "concat"), banks(3, "add")], ids=["n2-concat", "n3-add"])
def test_banked_step(bk, monkeypatch):
    """tfl_simulate_step with a banked model equals the operator sequence (1e-6) and oracle.simulate with the
    banked graph (2e-5, first step)."""
    from fluidnet_b200 import simulate
    monkeypatch.setattr(oracle.api, "model_forward", model_forward_banked)
    orc = oracle.Oracle()
    n = 24
    batch = make_batch((n, n, n), True, plume=True)
    mnp = synth.make_model(True, banks=bk)
    gm = make_gpu(mnp)
    mconf = oracle.default_mconf(dt=0.1, maccormackStrength=0.6, buoyancyScale=2.0 * n / 128,
                                 vorticityConfinementAmp=3.0, simMethod="convnet")
    a = {k: torch.from_numpy(v.copy()).cuda() for k, v in batch.items()}
    b = {k: torch.from_numpy(v.copy()).cuda() for k, v in batch.items()}
    simulate.simulate(None, mconf, a, gm)
    simulate.simulate_fused(None, mconf, b, gm)
    oracle.simulate(orc, mconf, batch, mnp)
    for k in ("density", "UDiv", "pDiv"):
        close(b[k].cpu().numpy(), a[k].cpu().numpy(), 1e-6, "fused vs ops " + k)
        close(b[k].cpu().numpy(), batch[k], 2e-5, "fused vs oracle " + k)


def test_banked_step_as_cuda_graph():
    """The fused step with a banked model captured once and replayed gives the bits of the direct call."""
    from fluidnet_b200 import simulate
    n = 32
    batch = make_batch((n, n, n), True, plume=True)
    gm = make_gpu(synth.make_model(True, banks=banks(2, "concat")))
    mconf = oracle.default_mconf(dt=0.1, maccormackStrength=0.6, buoyancyScale=2.0 * n / 128,
                                 vorticityConfinementAmp=3.0, simMethod="convnet")
    ga = {k: torch.from_numpy(v.copy()).cuda() for k, v in batch.items()}
    gb = {k: torch.from_numpy(v.copy()).cuda() for k, v in batch.items()}
    stream = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(stream):
        simulate.simulate_fused(None, mconf, ga, gm)
        simulate.simulate_fused(None, mconf, gb, gm)
        graph = simulate.StepGraph(mconf, gb, gm)
        for _ in range(2):
            simulate.simulate_fused(None, mconf, ga, gm)
            graph.launch()
        stream.synchronize()
        for k in ("density", "UDiv", "pDiv"):
            assert torch.equal(ga[k].view(torch.int32), gb[k].view(torch.int32)), k
        graph.close()


def test_banked_errors():
    # grid not divisible by 2^(N-1) at the split
    gm = make_gpu(synth.make_model(True, banks=banks(3, "concat")))
    f = torch.ones(1, 1, 8, 8, 10, device="cuda")
    with pytest.raises(TflError, match="divisible"):
        gm.forward((torch.zeros_like(f), torch.zeros(1, 3, 8, 8, 10, device="cuda"), f))
    gm2 = make_gpu(synth.make_model(False, banks=banks(2, "add")))
    f = torch.ones(1, 1, 1, 9, 8, device="cuda")
    with pytest.raises(TflError, match="divisible"):
        gm2.forward((torch.zeros_like(f), torch.zeros(1, 2, 1, 9, 8, device="cuda"), f))
    # the model.lua assertions on split / join / num
    layers = synth.make_model(True, banks=banks(2, "concat"))["layers"]
    for bk, msg in ((banks(0, "concat"), "banksNum >= 1"), (banks(2, "concat", 3, 3), "banksSplitStage < banksJoinStage"),
                    (banks(2, "concat", 0, 3), "banksSplitStage >= 1"), (banks(2, "concat", 1, 5), "banksJoinStage >= 1")):
        with pytest.raises(TflError, match=msg):
            fmodel.ProjectionModel(layers, True, banks=bk)
    # concat needs N x the channels at the join stage: an 'add' model's weights given as 'concat'
    add_layers = synth.make_model(True, banks=banks(2, "add"))["layers"]
    with pytest.raises(TflError, match="concatenates 2 banks"):
        fmodel.ProjectionModel(add_layers, True, banks=banks(2, "concat"))
    # the tensor-core modes cover the 3-D 'default' graph with banks split at stage 1 and joined at stage 3
    other = make_gpu(synth.make_model(True, banks=banks(2, "concat", 2, 4)))
    assert other.get_mode() == "fp32"
    for mode in ("tf32", "tf32x3"):
        with pytest.raises(TflError, match="split at stage 1 and joined at stage 3"):
            other.set_mode(mode)
    assert other.get_mode() == "fp32"
    gm.set_mode("fp32")                         # the fp32 path refuses the grid too
    f = torch.ones(1, 1, 8, 8, 10, device="cuda")
    with pytest.raises(TflError, match="divisible"):
        gm.forward((torch.zeros_like(f), torch.zeros(1, 3, 8, 8, 10, device="cuda"), f))
    # the z-slab path refuses a banked model
    lib, ctx = gm.ctx.lib, gm.ctx
    g = torch.zeros(1, 1, 8, 8, 8, device="cuda")
    from fluidnet_b200 import tfluids
    rc = lib.tfl_cnn_project_from_sums(ctx.h, gm.h, tfluids._grid(g), tfluids._grid(torch.zeros(1, 3, 8, 8, 8, device="cuda")),
                                       tfluids._grid(g), C.c_void_p(0), tfluids._grid(g),
                                       tfluids._grid(torch.zeros(1, 3, 8, 8, 8, device="cuda")), C.c_float(1e-5))
    assert rc != 0 and b"z-slab" in lib.tfl_last_error(ctx.h)


def write_mconf(path, mconf):
    from test_torch7_reader import W
    wr = W()

    def value(v):
        if isinstance(v, bool):
            return lambda: wr.boolean(v)
        if isinstance(v, (int, float)):
            return lambda: wr.number(v)
        if isinstance(v, str):
            return lambda: wr.string(v)
        return lambda: wr.table([(k, value(x)) for k, x in v.items()])

    value(mconf)()
    path.write_bytes(bytes(wr.b))


@pytest.mark.parametrize("agg", ["concat", "add"])
def test_banked_reference_file_end_to_end(tmp_path, agg):
    """A banked nngraph file and its mconf through ProjectionModel.from_reference_file: the model it builds runs and
    matches the CPU restatement of the synthesized model."""
    from test_torch7_banks import graph_nodes, mconf_of, write_graph
    mnp = synth.make_model(True, banks=banks(2, agg))
    write_graph(tmp_path / "net", graph_nodes(mnp), True)
    write_mconf(tmp_path / "net_mconf.bin", mconf_of(True, banksNum=2, banksAggregateMethod=agg))
    gm, mconf = fmodel.ProjectionModel.from_reference_file(str(tmp_path / "net"))
    assert mconf["banksNum"] == 2 and gm.banks == banks(2, agg) and gm.get_mode() == "tf32x3"
    batch = make_batch((8, 12, 16), True, nb=1)
    p0, inp = inputs_of(batch)
    wp, wU, _ = model_forward_banked(oracle.Oracle(), mnp, p0, batch["UDiv"], batch["flags"])
    gp, gU = gm.forward(inp)
    close(gp.cpu().numpy(), wp, 2e-5, "p")
    close(gU.cpu().numpy(), wU, 2e-5, "U")


@pytest.mark.parametrize("mode", ["tf32x3", "fp32"])
def test_banked_host_buffer_step(mode):
    """tfl_host_sim_step with a banked model returns what tfl_simulate_step leaves on the device."""
    from fluidnet_b200 import simulate, tfluids
    n = 16
    batch = make_batch((n, n, n), True, plume=True)
    gm = make_gpu(synth.make_model(True, banks=banks(2, "concat")))
    gm.set_mode(mode)
    mconf = oracle.default_mconf(dt=0.1, maccormackStrength=0.6, buoyancyScale=2.0 * n / 128,
                                 vorticityConfinementAmp=3.0, simMethod="convnet")
    dev_batch = {k: torch.from_numpy(v.copy()).cuda() for k, v in batch.items()}
    ctx = tfluids.context()
    lib = ctx.lib
    hs = C.c_void_p()
    keep = [np.ascontiguousarray(batch[k]) for k in ("flags", "UBC", "UBCInvMask", "densityBC", "densityBCInvMask")]
    ctx.check(lib.tfl_host_sim_create(ctx.h, 1, n, n, n, 1, *[a.ctypes.data for a in keep], C.byref(hs)))
    hp = torch.from_numpy(batch["pDiv"].copy()).pin_memory()
    hU = torch.from_numpy(batch["UDiv"].copy()).pin_memory()
    hd = torch.from_numpy(batch["density"].copy()).pin_memory()
    mc = simulate.make_mconf(mconf)
    try:
        for step in range(2):
            simulate.simulate_fused(None, mconf, dev_batch, gm)
            ctx.check(lib.tfl_host_sim_step(ctx.h, hs, hp.data_ptr(), hU.data_ptr(), hd.data_ptr(), C.byref(mc), gm.h))
            for k, h in (("density", hd), ("UDiv", hU), ("pDiv", hp)):
                close(h.numpy(), dev_batch[k].cpu().numpy(), 1e-6, "step %d %s" % (step, k))
    finally:
        lib.tfl_host_sim_destroy(ctx.h, hs)
