"""Dilated banks of the projection network (banksType 'dilate', lib/model.lua:252-361, lib/model_utils.lua:122-146) on
the GPU, on whole grids: the fp32 path for every graph, the tensor cores (3xTF32 by default, TF32) for the 3-D
'default' graph with banks split at stage 1 and joined at stage 3, where bank i runs as ordinary 3x3x3 layers on its
phase sub-grids.

  * Each dilated tensor-core layer through the test hook tfl_debug_conv3_tc_dilated (phase copy -> the existing layer
    kernel -> re-zeroing of short phases -> gather) against conv3d(dilation=d) in float64, per voxel within kappa S
    (the bound of tests/test_gpu_conv_tc.py: kappa = 2^-16 for 3xTF32, 2^-8 for TF32); nothing outside the interior
    of the output is written.
  * The dilated fp32 convolution, one launch through the test hook tfl_debug_conv_fp32_dilated, against conv3d /
    conv2d(dilation=d) in float64: per value within gamma_n S (the bound of tests/test_gpu_conv_fp32.py, whose
    argument does not depend on where the taps sit), exactly on the 2^-k 'exact' inputs, the generic kernel equal to
    the direct one bit for bit, nothing written outside the output.
  * model:forward against the CPU restatement (tests/dilate_oracle.py, pinned on torch.nn.functional by
    tests/test_oracle_model_dilate.py) within 2e-5 of each entry's max, on every graph; N = 1 'dilate' equals the
    single-bank model bit for bit; batch entries equal their own forward bit for bit.
  * The step against the operator sequence (1e-6) and oracle.simulate with the restated network (2e-5), step-graph
    replay, refusal of a stale graph, the host-buffer step; the tensor-core modes and the z-slab entry points refuse
    the model by name; a dilated reference file end to end."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import oracle
from dilate_oracle import model_forward_dilated
from fluidnet_b200 import synth
from fluidnet_b200 import model as fmodel
from fluidnet_b200._lib import TflError
from test_gpu_cnn_banks import close, inputs_of, make_batch, write_mconf
from test_gpu_step_paths import contexts  # noqa: F401  (fixture: library contexts of one test)
from test_gpu_conv_fp32 import (DIRECT, GENERIC, SIGMOID_ULPS, activate, check_guards, gamma, guarded, make_conv,
                                quantised_batch, seed_of, shuffle_model)

pytestmark = pytest.mark.gpu


def dilate(num, agg, s=1, j=3):
    return {"num": num, "split_stage": s, "join_stage": j, "aggregate": agg, "type": "dilate"}


def make_gpu(mnp, threshold=1e-5):
    return fmodel.ProjectionModel(mnp["layers"], mnp["is3D"], normalizeInputThreshold=threshold, pool=mnp.get("pool"),
                                  up=mnp.get("up"), poolType=mnp.get("poolType", "avg"),
                                  nonlinType=mnp.get("nonlinType", "relu"), banks=mnp.get("banks"))


# ---------------------------------------------------------------------------------------------------------------
# One dilated convolution
# ---------------------------------------------------------------------------------------------------------------
def conv_f64(x, w, b, d):
    kz, k = w.shape[2], w.shape[4]
    pad = (d * (kz - 1) // 2, d * (k - 1) // 2, d * (k - 1) // 2)
    dil = (d if kz > 1 else 1, d, d)
    return F.conv3d(torch.from_numpy(x).double(), torch.from_numpy(w).double(), torch.from_numpy(b).double(),
                    padding=pad, dilation=dil).numpy()


def run_conv(x, w, b, act, is3d, generic, d, what):
    from fluidnet_b200 import tfluids
    lib = tfluids.context().lib
    lib.tfl_debug_conv_fp32_dilated.argtypes = [C.c_void_p] * 5 + [C.c_int] * 11 + [C.POINTER(C.c_int32)]
    nb, cin, nz, ny, nx = x.shape
    cout, k = w.shape[0], w.shape[4]
    n = nb * cout * nz * ny * nx
    din = torch.from_numpy(x).cuda()
    buf, out = guarded(n)
    kernel = C.c_int32(0)
    ctx = tfluids._ctx_for(din)
    ctx.check(lib.tfl_debug_conv_fp32_dilated(ctx.h, din.data_ptr(), out.data_ptr(), w.ctypes.data, b.ctypes.data,
                                              cin, cout, k, act, int(is3d), nb, nz, ny, nx, generic, d,
                                              C.byref(kernel)))
    assert np.array_equal(din.cpu().numpy().view(np.uint32), x.view(np.uint32)), "%s: wrote its input" % what
    return check_guards(buf, n, what).reshape(nb, cout, nz, ny, nx), kernel.value


# (cout, k, is3d, grid, cin, kernel launch_conv_direct runs): the 'default' layers, 'tog''s k 5 and a generic shape;
# grids with axes d does not divide and axes shorter than d.
CONV_CASES = {
    "c8k3-3d": (8, 3, True, (5, 9, 37), 3, DIRECT),
    "c8k3-3d-cin8": (8, 3, True, (6, 7, 11), 8, DIRECT),
    "c16k3-2d": (16, 3, False, (1, 13, 37), 16, DIRECT),
    "c16k5-2d": (16, 5, False, (1, 19, 23), 3, DIRECT),
    "c6k3-3d": (6, 3, True, (3, 10, 12), 3, DIRECT),
    "c8k5-3d-generic": (8, 5, True, (5, 6, 13), 3, GENERIC),
}


@pytest.mark.parametrize("d", [2, 4, 8])
@pytest.mark.parametrize("case", list(CONV_CASES))
def test_dilated_convolution(case, d):
    cout, k, is3d, shape, cin, kernel = CONV_CASES[case]
    for inputs in ("exact", "signed", "nonneg"):
        for act in (0, 1, 2):
            what = "%s d%d %s act%d" % (case, d, inputs, act)
            x, w, b = make_conv(inputs, cin, cout, k, is3d, shape, 2, seed_of(what))
            got, ran = run_conv(x, w, b, act, is3d, 0, d, what)
            assert ran == kernel, "%s: ran kernel %d, expected %d" % (what, ran, kernel)
            pre = conv_f64(x, w, b, d)
            S = conv_f64(np.abs(x), np.abs(w), np.abs(b), d)
            n = int(np.prod(w.shape[1:])) + 1
            E = np.zeros_like(S) if inputs == "exact" else gamma(n) * S
            ref = activate(pre, act)
            bound = E / 4 + SIGMOID_ULPS * ref if act == 2 else E
            err = np.abs(got.astype(np.float64) - ref)
            assert (err <= bound).all(), "%s: %d values over the bound" % (what, (err > bound).sum())
            gen, ran = run_conv(x, w, b, act, is3d, 1, d, what + " generic")
            assert ran == GENERIC
            assert np.array_equal(gen.view(np.uint32), got.view(np.uint32)), "%s: generic differs from direct" % what


def test_dilation_one_is_the_plain_kernel():
    """dil = 1 through the dilated hook gives the bits of tfl_debug_conv_fp32."""
    from test_gpu_conv_fp32 import run_conv as run_plain
    x, w, b = make_conv("signed", 3, 8, 3, True, (5, 6, 9), 2, 11)
    for generic in (0, 1):
        a, _ = run_conv(x, w, b, 1, True, generic, 1, "d1")
        p, _ = run_plain(x, w, b, 1, True, generic, "plain")
        assert np.array_equal(a.view(np.uint32), p.view(np.uint32))


# ---------------------------------------------------------------------------------------------------------------
# model:forward
# ---------------------------------------------------------------------------------------------------------------
# (is3d, model_type, banks, (nz, ny, nx), nb)
FORWARD = {
    "3d-n2-concat": (True, "default", dilate(2, "concat"), (7, 10, 29), 2),
    "3d-n2-add": (True, "default", dilate(2, "add"), (6, 9, 30), 2),
    "3d-n3-concat": (True, "default", dilate(3, "concat"), (8, 11, 21), 1),
    "3d-n4-add-d8-over-z": (True, "default", dilate(4, "add"), (5, 12, 17), 2),
    "3d-n8-concat": (True, "default", dilate(8, "concat"), (6, 9, 13), 1),
    "3d-n8-add": (True, "default", dilate(8, "add"), (6, 9, 13), 1),
    "3d-n3-s2j4-concat": (True, "default", dilate(3, "concat", 2, 4), (6, 10, 12), 2),
    "3d-yang-n2-add": (True, "yang", dilate(2, "add", 1, 2), (6, 8, 10), 1),
    "3d-tog-n2-concat": (True, "tog", dilate(2, "concat"), (16, 16, 24), 2),
    "2d-n2-concat": (False, "default", dilate(2, "concat"), (1, 36, 51), 2),
    "2d-n3-add": (False, "default", dilate(3, "add"), (1, 41, 35), 1),
    "2d-n4-concat-s2j4": (False, "default", dilate(4, "concat", 2, 4), (1, 27, 30), 2),
    "2d-yang-n3-concat-s2j3": (False, "yang", dilate(3, "concat", 2, 3), (1, 20, 18), 1),
    "2d-tog-n2-add": (False, "tog", dilate(2, "add"), (1, 32, 48), 2),
}


MODE_TOL = {"fp32": 2e-5, "tf32x3": 2e-5, "tf32": 3e-3}


def tc_covered(is3d, model_type, bk):
    return is3d and model_type == "default" and bk["split_stage"] == 1 and bk["join_stage"] == 3


@pytest.mark.parametrize("mode", ["default", "fp32", "tf32"])
@pytest.mark.parametrize("case", list(FORWARD))
def test_dilated_forward(case, mode):
    orc = oracle.Oracle()
    is3d, model_type, bk, shape, nb = FORWARD[case]
    covered = tc_covered(is3d, model_type, bk)
    if mode != "default" and not covered:
        pytest.skip("fp32 only: the default mode is the only mode")
    batch = make_batch(shape, is3d, nb=nb)
    mnp = synth.make_model(is3d, model_type=model_type, banks=bk)
    p0, inp = inputs_of(batch)
    wp, wU, wscale = model_forward_dilated(orc, mnp, p0, batch["UDiv"], batch["flags"])
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


# (nb, (nz, ny, nx), log2 d): ragged axes, d above an axis, nb 1..3, and sub-rows on both sides of the z-streaming
# kernel's 128-position limit (nx 256 -> 128 at d = 2, nx 258 -> 129: the box kernel).
TC_LAYER_CASES = {
    "d2-ragged": (2, (5, 7, 9), 1),
    "d4-ragged-nb3": (3, (6, 9, 11), 2),
    "d8-over-z": (1, (5, 12, 17), 3),
    "d8-over-all": (2, (3, 6, 7), 3),
    "d2-nx256": (1, (3, 4, 256), 1),
    "d2-nx258": (1, (3, 4, 258), 1),
}


@pytest.mark.parametrize("split", [1, 0], ids=["tf32x3", "tf32"])
@pytest.mark.parametrize("layer", ["l1", "l2"])
@pytest.mark.parametrize("case", list(TC_LAYER_CASES))
def test_dilated_tc_layer(case, layer, split):
    from fluidnet_b200 import tfluids
    from test_gpu_conv_tc import KAPPA, SENTINEL, layout, make_layer, pack, unpack
    nb, shape, sh = TC_LAYER_CASES[case]
    d = 1 << sh
    cin = 3 if layer == "l1" else 8
    nz, ny, nx = shape
    for inputs in ("signed", "nonneg", "scaled"):
        what = "%s %s split%d %s" % (case, layer, split, inputs)
        x, w, b, _ = make_layer(inputs, cin, False, shape, nb, seed_of(what))
        px, py = layout(nb, nz, ny, nx)
        din = torch.from_numpy(pack(x, px, py, fill_unused=np.nan)).cuda()
        out = torch.full((nb, 2, nz + 2, py, px, 4), float(SENTINEL), device="cuda")
        ctx = tfluids._ctx_for(din)
        lib = ctx.lib
        lib.tfl_debug_conv3_tc_dilated.argtypes = [C.c_void_p] * 5 + [C.c_int] * 7
        ctx.check(lib.tfl_debug_conv3_tc_dilated(ctx.h, din.data_ptr(), out.data_ptr(), w.ctypes.data, b.ctypes.data,
                                                 cin, split, nb, nz, ny, nx, sh))
        o = out.cpu().numpy()
        inner = np.zeros(o.shape, bool)
        inner[:, :, 1:nz + 1, 1:ny + 1, 1:nx + 1, :] = True
        assert (o[~inner] == SENTINEL).all(), "%s: stray writes outside the interior" % what
        got = unpack(o, nz, ny, nx)
        assert np.isfinite(got).all(), what
        wt, bt = torch.from_numpy(w).double(), torch.from_numpy(b).double()
        conv = lambda a, ww, bb: F.conv3d(torch.from_numpy(a).double(), ww, bb, padding=d, dilation=d).numpy()
        ref = np.maximum(conv(x, wt, bt), 0.0)
        S = conv(np.abs(x), wt.abs(), bt.abs())
        err = np.abs(got.astype(np.float64) - ref)
        bound = KAPPA[split] * S
        assert (err <= bound).all(), "%s: %d voxels over kappa S, worst err/S %.3g" % (
            what, (err > bound).sum(), (err / np.maximum(S, 1e-30)).max())


@pytest.mark.parametrize("is3d", [True, False], ids=["3d", "2d"])
def test_one_dilated_bank_is_the_single_bank_graph(is3d):
    shape = (8, 12, 16) if is3d else (1, 24, 20)
    batch = make_batch(shape, is3d, nb=2)
    plain = synth.make_model(is3d)
    one = dict(plain, banks=dilate(1, "concat"))
    _, inp = inputs_of(batch)
    a, b = make_gpu(plain), make_gpu(one)
    assert a.get_mode() == b.get_mode()
    for x, y in zip(a.forward(inp), b.forward(inp)):
        assert torch.equal(x.view(torch.int32), y.view(torch.int32))


BATCH_GRAPHS = {
    "3d-n3-concat": (True, "default", dilate(3, "concat"), (6, 10, 13)),
    "3d-n2-add": (True, "default", dilate(2, "add"), (5, 9, 12)),
    "2d-tog-n2-concat-s1j2": (False, "tog", dilate(2, "concat", 1, 2), (1, 32, 48)),
    "2d-n3-concat-s2j4": (False, "default", dilate(3, "concat", 2, 4), (1, 21, 30)),
}


@pytest.mark.parametrize("name", list(BATCH_GRAPHS))
def test_batch_entries_are_independent(name):
    """Entry b of a batch of three equals its own forward bit for bit: the banks' per-entry writes into their
    channel slots of the 'concat' join keep the entries apart."""
    is3d, model_type, bk, shape = BATCH_GRAPHS[name]
    mnp = synth.make_model(is3d, model_type=model_type, banks=bk)
    gm = make_gpu(mnp)
    arrays = quantised_batch(shape, is3d, 3, seed_of(name) % 10000)
    p3, U3 = (t.cpu().numpy() for t in gm.forward(tuple(torch.from_numpy(a).cuda() for a in arrays)))
    assert np.isfinite(p3).all() and np.abs(p3).max() > 0
    for b in range(3):
        one = tuple(torch.from_numpy(np.ascontiguousarray(a[b:b + 1])).cuda() for a in arrays)
        p1, U1 = (t.cpu().numpy() for t in gm.forward(one))
        assert np.array_equal(p3[b:b + 1].view(np.uint32), p1.view(np.uint32)), (name, b, "p")
        assert np.array_equal(U3[b:b + 1].view(np.uint32), U1.view(np.uint32)), (name, b, "U")


# ---------------------------------------------------------------------------------------------------------------
# The step
# ---------------------------------------------------------------------------------------------------------------
def step_mconf(n):
    return oracle.default_mconf(dt=0.1, maccormackStrength=0.6, buoyancyScale=2.0 * n / 128,
                                vorticityConfinementAmp=3.0, simMethod="convnet")


@pytest.mark.parametrize("bk", [dilate(2, "concat"), dilate(3, "add")], ids=["n2-concat", "n3-add"])
def test_dilated_step(bk, monkeypatch):
    from fluidnet_b200 import simulate
    monkeypatch.setattr(oracle.api, "model_forward", model_forward_dilated)
    orc = oracle.Oracle()
    n = 20
    batch = make_batch((n, n, n), True, plume=True)
    mnp = synth.make_model(True, banks=bk)
    gm = make_gpu(mnp)
    mconf = step_mconf(n)
    a = {k: torch.from_numpy(v.copy()).cuda() for k, v in batch.items()}
    b = {k: torch.from_numpy(v.copy()).cuda() for k, v in batch.items()}
    simulate.simulate(None, mconf, a, gm)
    simulate.simulate_fused(None, mconf, b, gm)
    oracle.simulate(orc, mconf, batch, mnp)
    for k in ("density", "UDiv", "pDiv"):
        close(b[k].cpu().numpy(), a[k].cpu().numpy(), 1e-6, "fused vs ops " + k)
        close(b[k].cpu().numpy(), batch[k], 2e-5, "fused vs oracle " + k)


def test_dilated_step_graph_replay_and_stale_refusal(contexts):
    """The step with a dilated model captured once replays the direct call's bits; after the model runs on a larger
    grid (which grows the scratch arena the graph captured) the graph is refused.  A context of its own, so that the
    arena starts at this step's size."""
    from fluidnet_b200 import simulate
    n = 24
    batch = make_batch((n, n, n), True, plume=True)
    contexts.use(contexts.new())
    gm = make_gpu(synth.make_model(True, banks=dilate(2, "concat")))
    contexts.models.append(gm)
    mconf = step_mconf(n)
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
        big = make_batch((40, 40, 40), True)
        _, inp = inputs_of(big)
        gm.forward(inp)
        with pytest.raises(TflError, match="stale graph"):
            graph.launch()
        graph.close()


@pytest.mark.parametrize("mode", ["tf32x3", "fp32"])
def test_dilated_host_buffer_step(mode):
    from fluidnet_b200 import simulate, tfluids
    n = 16
    batch = make_batch((n, n, n), True, plume=True)
    gm = make_gpu(synth.make_model(True, banks=dilate(2, "concat")))
    gm.set_mode(mode)
    mconf = step_mconf(n)
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


# ---------------------------------------------------------------------------------------------------------------
# Refusals and import
# ---------------------------------------------------------------------------------------------------------------
def test_dilated_refusals():
    gm = make_gpu(synth.make_model(True, banks=dilate(2, "concat")))
    assert gm.get_mode() == "tf32x3"
    other = make_gpu(synth.make_model(True, banks=dilate(2, "concat", 2, 4)))
    assert other.get_mode() == "fp32"
    with pytest.raises(TflError, match="split at stage 1 and joined at stage 3"):
        other.set_mode("tf32x3")
    # the z-slab entry point refuses the model before any launch, naming the bank type
    from fluidnet_b200 import tfluids
    lib, ctx = gm.ctx.lib, gm.ctx
    g = torch.zeros(1, 1, 8, 8, 8, device="cuda")
    U = torch.zeros(1, 3, 8, 8, 8, device="cuda")
    rc = lib.tfl_cnn_project_from_sums(ctx.h, gm.h, tfluids._grid(g), tfluids._grid(U), tfluids._grid(g),
                                       C.c_void_p(0), tfluids._grid(g), tfluids._grid(torch.zeros_like(U)),
                                       C.c_float(1e-5))
    assert rc != 0 and b"banksType 'dilate'" in lib.tfl_last_error(ctx.h)
    # upsampling in a dilated stage (lib/model_utils.lua:125): no mconf builds it, the C ABI can ask for it
    mnp = shuffle_model(True, 2)
    with pytest.raises(TflError, match="upsampling not supported for dilated convolutions"):
        fmodel.ProjectionModel(mnp["layers"], True, pool=mnp["pool"], up=mnp["up"], banks=dilate(2, "concat", 2, 3))
    mres = fmodel.ProjectionModel(mnp["layers"], True, pool=mnp["pool"], up=mnp["up"],
                                  banks=dict(dilate(2, "concat", 2, 3), type="mres"))
    assert mres.get_mode() == "fp32"
    # no divisibility requirement: a grid no dilation divides runs
    f = torch.ones(1, 1, 7, 9, 11, device="cuda")
    gm.forward((torch.zeros_like(f), torch.zeros(1, 3, 7, 9, 11, device="cuda"), f))


@pytest.mark.parametrize("agg", ["concat", "add"])
def test_dilated_reference_file_end_to_end(tmp_path, agg):
    from test_torch7_banks import mconf_of
    from test_torch7_dilate import write_dilated
    mnp = synth.make_model(True, banks=dilate(3, agg))
    write_dilated(tmp_path / "net", mnp, True)
    write_mconf(tmp_path / "net_mconf.bin", mconf_of(True, banksNum=3, banksAggregateMethod=agg, banksType="dilate"))
    gm, mconf = fmodel.ProjectionModel.from_reference_file(str(tmp_path / "net"))
    assert mconf["banksType"] == "dilate" and gm.banks == dilate(3, agg) and gm.get_mode() == "tf32x3"
    batch = make_batch((8, 12, 16), True, nb=1)
    p0, inp = inputs_of(batch)
    wp, wU, _ = model_forward_dilated(oracle.Oracle(), mnp, p0, batch["UDiv"], batch["flags"])
    gp, gU = gm.forward(inp)
    close(gp.cpu().numpy(), wp, 2e-5, "p")
    close(gU.cpu().numpy(), wU, 2e-5, "U")


def test_slab_step_refuses_dilated_banks():
    """tfl_slab_sim_step (cnn_slab_check) refuses a dilated model, in every mode, naming the bank type, before it
    launches anything."""
    from fluidnet_b200 import simulate
    from fluidnet_b200.slab import NativeSlabSimulator
    from test_gpu_slab_banks import _problem, _refused
    dev = torch.device("cuda", 0)
    tb, mconf, _ = _problem(32, 16, 16, None)
    sim = NativeSlabSimulator(tb, mconf, synth.make_model(True)["layers"], dev, rank=0, world=1, margin=6)
    ctx, mc = sim.ctx, simulate.make_mconf(mconf)
    gm = fmodel.ProjectionModel(synth.make_model(True, banks=dilate(2, "add"))["layers"], True, banks=dilate(2, "add"))
    for mode in ("tf32x3", "fp32"):
        gm.set_mode(mode)
        msg = _refused(ctx, lambda: ctx.lib.tfl_slab_sim_step(ctx.h, sim.h, C.byref(mc), gm.h))
        assert b"banksType 'dilate'" in msg, msg
