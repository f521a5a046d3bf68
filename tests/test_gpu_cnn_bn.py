"""Batch normalization (addBatchNorm) and nonlinType 'relu6' of the projection network on the GPU: the fp32 path
for every graph and the tensor cores (3xTF32 by default, TF32) for the 3-D 'default' single-bank graph (relu6 also
banked), with batch statistics (modules saved with train = true) and running statistics.

  * One tensor-core layer with BN through the test hook tfl_debug_conv3_tc_bn against float64: the running-statistics
    epilogue y = a act(h) + c within |a| kappa S + 2 u32 (|a act(h)| + |c|) (kappa S: the per-voxel bound of
    tests/test_gpu_conv_tc.py), and batch statistics of the layer's output (padded-layout statistics, finalize, apply
    on the interior) against the float64 statistics of the float64 layer; relu6; at nx <= 128 (z-streaming kernel) and
    nx > 128 (box kernel); the padded border and the planes outside the interior are never written.

  * The BN kernels (launch_bn_stats / _finalize / _apply) through the test hook tfl_debug_bn against float64.
    Bounds: the partial and final sums run in fp64 over N = nb n float32 values, so each of sum x and sum x^2 is off
    by at most N u64 times the sum of magnitudes (u64 = 2^-53); hence |d mean| <= N u64 mean|x| and
    |d var| <= 2 N u64 mean(x^2) + 2 |mean| |d mean| (var = E x^2 - mean^2 in fp64).  a = w invstd and
    c = b - mean a are each rounded once to float32, and y = fma(a, x, c) once more, so
    |y - y64| <= 2 u32 (|a| (|x| + |mean|) + |c| + |y64|) up to the (far smaller) fp64 terms, u32 = 2^-24.  The fp64
    sums are what keeps a channel with |mean| / std ~ 1e3 within these bounds; float32 sums of x^2 would lose var.
    A second call gives the same bits; a dead channel with eps = 0 gives exactly b; nothing outside the nb c n values
    (the gaps of a batch stride) is written.
  * model:forward against oracle.model_forward(f64=True) (pinned on torch.nn.functional by
    tests/test_oracle_model_bn.py) within 2e-5 of each entry's max (fp32, 3xTF32; 3e-3 TF32), on every graph, in both BN modes, nb = 1 and 2, relu6 with
    values past 6.  With batch
    statistics changing entry 1 changes entry 0; with running statistics it does not, bit for bit.  Running statistics
    with w = 1, b = 0, mean 0, var 1 - eps equal the model without BN.
  * The step: a BN model in 3xTF32 takes the fused step at any nb (fused_step_applies, restated as takes_fused_path
    in tests/test_gpu_step_paths.py; tests/test_gpu_batch_models.py steps BN models batched); here at nb = 1 it and matches the operator sequence (1e-6) and oracle.simulate with the restated
    network (2e-5); step-graph replay bit for bit; the host-buffer step.  The tensor-core modes refuse banked BN models
    and the z-slab entry points every BN model, by name; a BN reference file end to end."""
import ctypes as C

import numpy as np
import pytest
import torch

import oracle
from fluidnet_b200 import synth
from fluidnet_b200 import model as fmodel
from fluidnet_b200._lib import TflError
from scenes import banks, bn_model, close, inputs_of, plume_batch, step_mconf, to_gpu
from step_cases import MODE_TOL, contexts
from torch7_writer import write_mconf

pytestmark = pytest.mark.gpu

U32, U64 = 2.0 ** -24, 2.0 ** -53


# ---------------------------------------------------------------------------------------------------------------
# The BN kernels
# ---------------------------------------------------------------------------------------------------------------
def run_bn(x, c, n, bstride, w, b, eps):
    """x: [nb][bstride] float32 holding the [c][n] values of each entry first; returns (y, stats [c][2], ac [2][c])."""
    from fluidnet_b200 import tfluids
    lib = tfluids.context().lib
    lib.tfl_debug_bn.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int64, C.c_int64, C.c_void_p,
                                 C.c_void_p, C.c_float, C.c_void_p, C.c_void_p]
    dx = torch.from_numpy(x.copy()).cuda()
    stats = np.zeros((c, 2), np.float64)
    ac = np.zeros((2, c), np.float32)
    ctx = tfluids._ctx_for(dx)
    ctx.check(lib.tfl_debug_bn(ctx.h, dx.data_ptr(), x.shape[0], c, n, bstride,
                               None if w is None else w.ctypes.data, None if b is None else b.ctypes.data, eps,
                               stats.ctypes.data, ac.ctypes.data))
    return dx.cpu().numpy(), stats, ac


def bn_inputs(nb, c, n, gap, seed):
    rs = np.random.RandomState(seed)
    x = np.full((nb, c * n + gap), np.float32(-7.25), np.float32)          # gap: a sentinel between entries
    v = rs.randn(nb, c, n).astype(np.float32)
    v[:, 0] = np.maximum(v[:, 0], 0) * 3                                 # relu-like
    v[:, 1] = 0.0                                                        # dead channel
    v[:, 2] = np.float32(1e3) + v[:, 2]                                  # |mean| / std ~ 1e3
    v[:, 3] = rs.rand(nb, n).astype(np.float32) * 1e-3                   # tiny values
    x[:, :c * n] = v.reshape(nb, c * n)
    return x, v


@pytest.mark.parametrize("nb,n,gap", [(1, 1, 0), (2, 37 * 11, 0), (3, 4096 + 13, 64), (2, 130 * 129, 5)])
def test_bn_kernels_against_float64(nb, n, gap):
    c = 5
    x, v = bn_inputs(nb, c, n, gap, nb * 1000 + n)
    rs = np.random.RandomState(n)
    w = (0.5 + rs.rand(c)).astype(np.float32)
    b = (rs.rand(c) - 0.5).astype(np.float32)
    for eps, wb in ((1e-4, True), (0.0, True), (1e-5, False)):
        y, stats, ac = run_bn(x, c, n, c * n + gap, w if wb else None, b if wb else None, eps)
        y2, stats2, ac2 = run_bn(x, c, n, c * n + gap, w if wb else None, b if wb else None, eps)
        assert np.array_equal(y.view(np.uint32), y2.view(np.uint32)) and np.array_equal(stats, stats2)
        assert (y[:, c * n:] == np.float32(-7.25)).all(), "wrote outside the values"
        v64 = v.astype(np.float64)
        N = nb * n
        mean = v64.mean(axis=(0, 2))
        var = v64.var(axis=(0, 2))
        dmean = N * U64 * np.abs(v64).mean(axis=(0, 2)) + 1e-300
        dvar = 2 * N * U64 * (v64 ** 2).mean(axis=(0, 2)) + 2 * np.abs(mean) * dmean + 1e-300
        assert (np.abs(stats[:, 0] - mean) <= dmean).all(), (stats[:, 0], mean)
        assert (np.abs(stats[:, 1] - var) <= dvar).all(), (stats[:, 1], var)
        ww = w.astype(np.float64) if wb else np.ones(c)
        bb = b.astype(np.float64) if wb else np.zeros(c)
        ve = var + np.float64(np.float32(eps))
        invstd = np.where(ve == 0, 0.0, 1.0 / np.sqrt(np.where(ve == 0, 1.0, ve)))
        a64 = ww * invstd
        c64 = bb - mean * a64
        s = lambda t: t[None, :, None]
        y64 = s(a64) * v64 + s(c64)
        bound = 2 * U32 * (s(np.abs(a64)) * (np.abs(v64) + s(np.abs(mean))) + s(np.abs(c64)) + np.abs(y64)) + 1e-30
        got = y[:, :c * n].reshape(nb, c, n).astype(np.float64)
        assert (np.abs(got - y64) <= bound).all(), np.abs(got - y64).max()
        if eps == 0.0:
            assert (got[:, 1] == np.float32(bb[1])).all(), "dead channel with eps = 0 must give exactly b"


# ---------------------------------------------------------------------------------------------------------------
# model:forward
# ---------------------------------------------------------------------------------------------------------------
# (is3d, model_type, banks, inputs, (nz, ny, nx))
FORWARD = {
    "3d-default": (True, "default", None, None, (8, 10, 12)),
    "3d-default-skip-udiv": (True, "default", None, {"inputChannels": {"UDiv": True}, "addPressureSkip": True},
                             (7, 9, 11)),
    "3d-tog": (True, "tog", None, None, (16, 16, 24)),
    "3d-yang": (True, "yang", None, None, (6, 8, 10)),
    "3d-mres-n2-concat": (True, "default", banks(2, "concat", "mres"), None, (8, 12, 16)),
    "3d-mres-n3-add": (True, "default", banks(3, "add", "mres"), None, (8, 8, 12)),
    "3d-dilate-n2-concat": (True, "default", banks(2, "concat", "dilate"), None, (7, 10, 29)),
    "3d-dilate-n3-add-s2j4": (True, "default", banks(3, "add", "dilate", 2, 4), None, (6, 10, 12)),
    "2d-default": (False, "default", None, None, (1, 36, 51)),
    "2d-tog": (False, "tog", None, None, (1, 32, 48)),
    "2d-mres-n2-add": (False, "default", banks(2, "add", "mres"), None, (1, 32, 24)),
    "2d-dilate-n3-concat": (False, "default", banks(3, "concat", "dilate"), None, (1, 41, 35)),
}


def tc_covered(is3d, model_type, bk):
    """The tensor-core path takes BN on the single-bank 3-D 'default' graph (banked BN models run on fp32)."""
    return is3d and model_type == "default" and bk is None


@pytest.mark.parametrize("mode", ["default", "fp32", "tf32"])
@pytest.mark.parametrize("nb", [1, 2])
@pytest.mark.parametrize("variant", ["batch", "running", "batch-relu6-noaffine", "running-relu6"])
@pytest.mark.parametrize("case", list(FORWARD))
def test_bn_forward(case, variant, nb, mode):
    orc = oracle.Oracle()
    is3d, model_type, bk, inputs, shape = FORWARD[case]
    covered = tc_covered(is3d, model_type, bk)
    if mode != "default" and not covered:
        pytest.skip("fp32 only: the default mode is the only mode")
    relu6 = "relu6" in variant and model_type != "yang"
    mnp = bn_model(variant.startswith("batch"), is3d, model_type, bk, inputs, relu6, "noaffine" not in variant)
    batch = plume_batch(shape, is3d, nb=nb)
    p0, inp = inputs_of(batch)
    wp, wU, wscale = oracle.model_forward(orc, mnp, p0, batch["UDiv"], batch["flags"], f64=True)
    gm = fmodel.ProjectionModel.from_model(mnp)
    assert gm.get_mode() == ("tf32x3" if covered else "fp32")
    if mode != "default":
        gm.set_mode(mode)
    tol = MODE_TOL[gm.get_mode()]
    gp, gU = gm.forward(inp, return_scale=True)
    gp, gU = gp.cpu().numpy(), gU.cpu().numpy()
    for b in range(nb):
        assert abs(gm.last_scale[b] - wscale[b]) <= 1e-5 * wscale[b]
        close(gp[b], wp[b], tol, "p[%d]" % b)
        close(gU[b], wU[b], tol, "U[%d]" % b)


@pytest.mark.parametrize("mode", ["tf32x3", "tf32"])
@pytest.mark.parametrize("bk", [banks(2, "concat", "mres"), banks(3, "add", "dilate")],
                         ids=["mres-n2-concat", "dilate-n3-add"])
def test_relu6_banked_on_tensor_cores(bk, mode):
    """relu6 without BN keeps the banked tensor-core path: the clamp is in the bank layers' and the join's epilogues."""
    mnp = synth.make_model(True, banks=bk)
    mnp["nonlinType"] = "relu6"
    mnp["layers"][0][0][0][...] *= np.float32(30.0)
    batch = plume_batch((8, 12, 16), True, nb=2)
    p0, inp = inputs_of(batch)
    wp, wU, _ = oracle.model_forward(oracle.Oracle(), mnp, p0, batch["UDiv"], batch["flags"], f64=True)
    gm = fmodel.ProjectionModel.from_model(mnp)
    assert gm.get_mode() == "tf32x3"
    gm.set_mode(mode)
    gp, gU = gm.forward(inp)
    close(gp.cpu().numpy(), wp, MODE_TOL[mode], "p")
    close(gU.cpu().numpy(), wU, MODE_TOL[mode], "U")


# (nb, (nz, ny, nx)): tile and grid edges of the z-streaming kernel (nx <= 128) and the box kernel (nx > 128)
TC_BN_CASES = {"ragged": (2, (5, 7, 9)), "nx128": (1, (3, 5, 128)), "nx130": (1, (3, 4, 130)), "nb3": (3, (4, 6, 33))}


@pytest.mark.parametrize("split", [1, 0], ids=["tf32x3", "tf32"])
@pytest.mark.parametrize("relu6", [0, 1])
@pytest.mark.parametrize("case", list(TC_BN_CASES))
def test_tc_bn_layer(case, relu6, split):
    import torch.nn.functional as F
    from fluidnet_b200 import tfluids
    from tc_conv import KAPPA, SENTINEL, layout, make_layer, pack, unpack
    nb, shape = TC_BN_CASES[case]
    nz, ny, nx = shape
    kappa = KAPPA[split]
    for cin in (3, 8):
        what = "%s cin%d relu6=%d split%d" % (case, cin, relu6, split)
        x, w, b, _ = make_layer("signed", cin, False, shape, nb, nb * 100 + nx + cin)
        x *= np.float32(8.0 if relu6 else 1.0)               # values past 6 after the layer
        w *= np.float32(4.0)
        rs = np.random.RandomState(nx)
        ep = np.concatenate([(0.5 + rs.rand(8)), rs.rand(8) - 0.5]).astype(np.float32)
        bw, bb = (0.5 + rs.rand(8)).astype(np.float32), (rs.rand(8) - 0.5).astype(np.float32)
        px, py = layout(nb, nz, ny, nx)
        din = torch.from_numpy(pack(x, px, py)).cuda()
        ctx = tfluids._ctx_for(din)
        lib = ctx.lib
        lib.tfl_debug_conv3_tc_bn.argtypes = [C.c_void_p] * 5 + [C.c_int] * 3 + [C.c_void_p, C.c_int, C.c_void_p,
                                                                                  C.c_void_p, C.c_float, C.c_void_p,
                                                                                  C.c_void_p] + [C.c_int] * 4
        wt, bt = torch.from_numpy(w).double(), torch.from_numpy(b).double()
        conv = lambda a, ww, bbb: F.conv3d(torch.from_numpy(a).double(), ww, bbb, padding=1).numpy()
        pre = conv(x, wt, bt)
        S = conv(np.abs(x), wt.abs(), bt.abs())
        h64 = np.minimum(np.maximum(pre, 0), 6) if relu6 else np.maximum(pre, 0)
        s = lambda t: t[None, :, None, None, None]
        for batch_mode in (0, 1):
            out = torch.full((nb, 2, nz + 2, py, px, 4), float(SENTINEL), device="cuda")
            stats = np.zeros(16, np.float64)
            ac = np.zeros(16, np.float32)
            ctx.check(lib.tfl_debug_conv3_tc_bn(ctx.h, din.data_ptr(), out.data_ptr(), w.ctypes.data, b.ctypes.data,
                                                cin, split, relu6, None if batch_mode else ep.ctypes.data, batch_mode,
                                                bw.ctypes.data, bb.ctypes.data, 1e-4, stats.ctypes.data, ac.ctypes.data,
                                                nb, nz, ny, nx))
            o = out.cpu().numpy()
            inner = np.zeros(o.shape, bool)
            inner[:, :, 1:nz + 1, 1:ny + 1, 1:nx + 1, :] = True
            assert (o[~inner] == SENTINEL).all(), "%s batch=%d: writes outside the interior" % (what, batch_mode)
            got = unpack(o, nz, ny, nx).astype(np.float64)
            if not batch_mode:
                a, c = ep[:8].astype(np.float64), ep[8:].astype(np.float64)
                ref = s(a) * h64 + s(c)
                bound = s(np.abs(a)) * kappa * S + 2 * U32 * (np.abs(s(a) * h64) + s(np.abs(c))) + 1e-30
            else:
                mean = h64.mean(axis=(0, 2, 3, 4))
                var = h64.var(axis=(0, 2, 3, 4))
                E = kappa * S
                dmean = E.mean(axis=(0, 2, 3, 4)) + 1e-12 * (np.abs(mean) + 1)
                dvar = 2 * (np.abs(h64 - s(mean)) * E).mean(axis=(0, 2, 3, 4)) + E.max() ** 2 + 1e-10 * (var + 1)
                st = stats.reshape(8, 2)
                assert (np.abs(st[:, 0] - mean) <= dmean).all(), (what, st[:, 0], mean)
                assert (np.abs(st[:, 1] - var) <= dvar).all(), (what, st[:, 1], var)
                a, c = ac[:8].astype(np.float64), ac[8:].astype(np.float64)
                ref = s(a) * h64 + s(c)
                bound = s(np.abs(a)) * E + 2 * U32 * (np.abs(s(a) * h64) + s(np.abs(c))) + 1e-30
            err = np.abs(got - ref)
            assert (err <= bound).all(), "%s batch=%d: %d voxels over the bound, worst %.3g" % (
                what, batch_mode, (err > bound).sum(), (err / bound).max())


@pytest.mark.parametrize("case", ["3d-default", "3d-mres-n2-concat", "3d-dilate-n2-concat", "2d-tog"])
def test_batch_statistics_couple_the_entries(case):
    is3d, model_type, bk, inputs, shape = FORWARD[case]
    batch = plume_batch(shape, is3d, nb=2)
    p0, inp = inputs_of(batch)
    other = list(t.clone() for t in inp)
    other[1][1] *= 2.0                  # entry 1's velocity
    for train in (True, False):
        gm = fmodel.ProjectionModel.from_model(bn_model(train, is3d, model_type, bk, inputs))
        a = gm.forward(tuple(inp))[0][0].cpu().numpy()
        b = gm.forward(tuple(other))[0][0].cpu().numpy()
        if train:
            assert not np.array_equal(a, b), "batch statistics: entry 0 must depend on entry 1"
        else:
            assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), "running statistics couple the entries"


@pytest.mark.parametrize("is3d", [True, False], ids=["3d", "2d"])
def test_identity_running_statistics_equal_the_model_without_bn(is3d):
    mnp = synth.make_model(is3d, batch_norm={"train": False})
    for e in mnp["batchNorm"]["layers"]:
        c = len(e["running_mean"])
        e.update(weight=np.ones(c, np.float32), bias=np.zeros(c, np.float32), running_mean=np.zeros(c, np.float32),
                 running_var=np.full(c, 1.0 - 1e-4, np.float32), eps=1e-4)
    batch = plume_batch((8, 10, 12) if is3d else (1, 30, 26), is3d, nb=2)
    _, inp = inputs_of(batch)
    plain = fmodel.ProjectionModel.from_model(dict(mnp, batchNorm=None))
    plain.set_mode("fp32")
    with_bn = fmodel.ProjectionModel.from_model(mnp)
    with_bn.set_mode("fp32")
    for x, y in zip(with_bn.forward(inp), plain.forward(inp)):
        close(x.cpu().numpy(), y.cpu().numpy(), 2e-5, "identity BN")


# ---------------------------------------------------------------------------------------------------------------
# The step
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("train", [True, False], ids=["batch", "running"])
def test_bn_step(train, contexts):
    from fluidnet_b200 import simulate
    orc = oracle.Oracle()
    n = 20
    batch = plume_batch((n, n, n), True, inflow=n / 128.0 * 4)
    from step_cases import takes_fused_path
    mnp = bn_model(train, relu6=True)
    contexts.use(contexts.new())
    gm = fmodel.ProjectionModel.from_model(mnp)
    contexts.models.append(gm)
    assert gm.get_mode() == "tf32x3" and takes_fused_path({"mode": gm.get_mode(), "nb": 1, "pbc": False})
    mconf = step_mconf(n)
    a = to_gpu(batch)
    b = to_gpu(batch)
    g = to_gpu(batch)
    simulate.simulate(None, mconf, a, gm)
    simulate.simulate_fused(None, mconf, b, gm)
    oracle.simulate(orc, mconf, batch, mnp, f64=True)
    for k in ("density", "UDiv", "pDiv"):
        close(b[k].cpu().numpy(), a[k].cpu().numpy(), 1e-6, "step vs ops " + k)
        close(b[k].cpu().numpy(), batch[k], 2e-5, "step vs oracle " + k)
    stream = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(stream):
        simulate.simulate_fused(None, mconf, g, gm)          # g now holds b's state
        graph = simulate.StepGraph(mconf, g, gm)
        for _ in range(2):
            simulate.simulate_fused(None, mconf, b, gm)
            graph.launch()
        stream.synchronize()
        graph.close()
    for k in ("density", "UDiv", "pDiv"):
        assert torch.equal(b[k].view(torch.int32), g[k].view(torch.int32)), "graph replay " + k


def test_bn_host_buffer_step():
    from fluidnet_b200 import simulate, tfluids
    n = 16
    batch = plume_batch((n, n, n), True, inflow=n / 128.0 * 4)
    gm = fmodel.ProjectionModel.from_model(bn_model(True))
    mconf = step_mconf(n)
    dev_batch = to_gpu(batch)
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
def test_bn_refusals():
    from fluidnet_b200 import tfluids
    gm = fmodel.ProjectionModel.from_model(bn_model(True))
    assert gm.get_mode() == "tf32x3"
    for bk in (banks(2, "concat", "mres"), banks(2, "add", "dilate")):
        banked = fmodel.ProjectionModel.from_model(bn_model(False, bk=bk))
        assert banked.get_mode() == "fp32"
        with pytest.raises(TflError, match="batch normalization"):
            banked.set_mode("tf32")
    lib, ctx = gm.ctx.lib, gm.ctx
    g = torch.zeros(1, 1, 8, 8, 8, device="cuda")
    U = torch.zeros(1, 3, 8, 8, 8, device="cuda")
    rc = lib.tfl_cnn_project_from_sums(ctx.h, gm.h, tfluids._grid(g), tfluids._grid(U), tfluids._grid(g),
                                       C.c_void_p(0), tfluids._grid(g), tfluids._grid(torch.zeros_like(U)),
                                       C.c_float(1e-5))
    assert rc != 0 and b"batch normalization" in lib.tfl_last_error(ctx.h)
    mnp = bn_model(True)
    bad = dict(mnp["batchNorm"], layers=[dict(e) for e in mnp["batchNorm"]["layers"]])
    bad["layers"][2]["eps"] = -1e-4
    with pytest.raises(TflError, match="eps"):
        fmodel.ProjectionModel.from_model(dict(mnp, batchNorm=bad))
    sig = synth.make_model(True, model_type="yang")
    lib2 = gm.ctx.lib
    from fluidnet_b200 import _lib
    norm = _lib.CnnNorm(1, 0, 0, None, None)
    h = C.c_void_p()
    w, b = zip(*sig["layers"])
    wp = (C.POINTER(C.c_float) * 4)(*[a.ctypes.data_as(C.POINTER(C.c_float)) for a in w])
    bp = (C.POINTER(C.c_float) * 4)(*[a.ctypes.data_as(C.POINTER(C.c_float)) for a in b])
    ints = lambda v: (C.c_int32 * 4)(*v)
    rc = lib2.tfl_cnn_create_model_norm(ctx.h, 1, 4, ints([3, 6, 6, 6]), ints([6, 6, 6, 1]), ints([3, 1, 1, 1]), None,
                                        None, 0, 1, None, None, C.byref(norm), wp, bp, C.byref(h))
    assert rc != 0 and b"relu6" in lib2.tfl_last_error(ctx.h) and b"sigmoid" in lib2.tfl_last_error(ctx.h)
    norm = _lib.CnnNorm(0, 1, 1, None, None)
    rc = lib2.tfl_cnn_create_model_norm(ctx.h, 1, 4, ints([3, 6, 6, 6]), ints([6, 6, 6, 1]), ints([3, 1, 1, 1]), None,
                                        None, 0, 0, None, None, C.byref(norm), wp, bp, C.byref(h))
    assert rc != 0 and b"addBatchNorm" in lib2.tfl_last_error(ctx.h)


def test_slab_step_refuses_bn():
    from fluidnet_b200 import simulate
    from fluidnet_b200.slab import NativeSlabSimulator
    from slab_cases import banked_problem, refused
    dev = torch.device("cuda", 0)
    tb, mconf, _ = banked_problem(32, 16, 16, None)
    sim = NativeSlabSimulator(tb, mconf, synth.make_model(True)["layers"], dev, rank=0, world=1, margin=6)
    ctx, mc = sim.ctx, simulate.make_mconf(mconf)
    for train in (True, False):
        gm = fmodel.ProjectionModel.from_model(bn_model(train))
        msg = refused(ctx, lambda: ctx.lib.tfl_slab_sim_step(ctx.h, sim.h, C.byref(mc), gm.h))
        assert b"batch normalization" in msg, msg


@pytest.mark.parametrize("train", [True, False])
def test_bn_reference_file_end_to_end(tmp_path, train):
    from torch7_writer import bn_graph, mconf_for, write_bn_graph
    bk = banks(2, "concat", "mres")
    mnp = bn_model(train, bk={k: v for k, v in bk.items() if k != "type"})
    write_bn_graph(tmp_path / "net", bn_graph(mnp, True, train=train, interleave=True), True)
    write_mconf(tmp_path / "net_mconf.bin", mconf_for(True, bk, True))
    gm, mconf = fmodel.ProjectionModel.from_reference_file(str(tmp_path / "net"))
    assert mconf["addBatchNorm"] and gm.get_mode() == "fp32"          # banked: the fp32 path
    batch = plume_batch((8, 12, 16), True, nb=2)
    p0, inp = inputs_of(batch)
    wp, wU, _ = oracle.model_forward(oracle.Oracle(), mnp, p0, batch["UDiv"], batch["flags"], f64=True)
    gp, gU = gm.forward(inp)
    close(gp.cpu().numpy(), wp, 2e-5, "p")
    close(gU.cpu().numpy(), wU, 2e-5, "U")
