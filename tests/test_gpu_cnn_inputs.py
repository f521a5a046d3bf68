"""The input block of the projection network (lib/model.lua:27-150, :357-387: inputChannels, normalizeInput,
normalizeInputFunc, normalizeInputChan, addPressureSkip) on the GPU: model:forward against the CPU restatement
(oracle.model_forward, pinned on torch.nn.functional by tests/test_oracle_model_inputs.py), the returned scale,
the default block built by every creator bit for bit, layer 1 and the bank pyramid on the two-plane
tensor-core input, the step and its graph, and the z-slab refusal.

Tolerances as tests/test_gpu_cnn_banks.py: p and U within 2e-5 (fp32, 3xTF32) or 3e-3 (TF32) of each entry's max,
the zero pattern of U exact; the scale within 1e-6 relative."""
import ctypes as C

import numpy as np
import pytest
import torch

import oracle
from fluidnet_b200 import model as fmodel
from fluidnet_b200 import synth
from oracle.model import model_input
from scenes import banks, close, inputs_of, plume_batch, step_mconf, to_gpu
from slab_cases import banked_problem, refused
from step_cases import MODE_TOL
from tc_conv import SENTINEL, check_layer, is_sentinel, layout, make_layer, pack, unpack

pytestmark = pytest.mark.gpu

ALL = dict(pDiv=True, UDiv=True, div=True, flags=True)
U_ONLY = dict(pDiv=False, UDiv=True, div=False, flags=True)
P_U = dict(pDiv=True, UDiv=True, div=False, flags=True)
DIV_ONLY = dict(pDiv=False, UDiv=False, div=True, flags=True)

def ins(ch=None, **kw):
    return dict(inputChannels=ch or dict(pDiv=True, UDiv=False, div=True, flags=True), **kw)


# (is3d, model_type, banks, inputs, (nz, ny, nx), nb).  The first group runs on the fp32 path only ('yang', 'tog',
# 2-D, banks not split 1 / joined 3); the second is the 3-D 'default' graph the tensor cores cover.
FP32 = {
    "2d-all-divchan-skip": (False, "default", None, ins(ALL, normalizeInputChan="div", addPressureSkip=True),
                            (1, 20, 26), 2),
    "2d-div-pchan": (False, "default", None, ins(DIV_ONLY, normalizeInputChan="pDiv"), (1, 18, 22), 1),
    "3d-yang-skip-norm-pchan": (True, "yang", None, ins(addPressureSkip=True, normalizeInputFunc="norm",
                                                        normalizeInputChan="pDiv"), (6, 8, 10), 2),
    "2d-yang-skip-unnormalized": (False, "yang", None, ins(addPressureSkip=True, normalizeInput=False), (1, 16, 20), 1),
    "3d-tog-all": (True, "tog", None, ins(ALL), (16, 16, 24), 1),
    "2d-tog-pU-pchan": (False, "tog", None, ins(P_U, normalizeInputChan="pDiv"), (1, 32, 48), 2),
    "2d-n2-concat-U-skip": (False, "default", banks(2, "concat"), ins(U_ONLY, addPressureSkip=True), (1, 36, 52), 2),
    "3d-yang-n2-add-norm-divchan": (True, "yang", banks(2, "add", s=1, j=2), ins(normalizeInputFunc="norm",
                                                                            normalizeInputChan="div"), (6, 8, 10), 1),
    "3d-n2-concat-s2j4-all": (True, "default", banks(2, "concat", s=2, j=4), ins(ALL), (6, 10, 12), 2),
}
TC = {
    "3d-U-norm": (True, "default", None, ins(U_ONLY, normalizeInputFunc="norm"), (6, 10, 14), 2),
    "3d-all-skip": (True, "default", None, ins(ALL, addPressureSkip=True), (7, 9, 31), 2),
    "3d-U-norm-skip": (True, "default", None, ins(U_ONLY, normalizeInputFunc="norm", addPressureSkip=True),
                       (5, 12, 34), 1),
    "3d-pU-pchan": (True, "default", None, ins(P_U, normalizeInputChan="pDiv"), (6, 8, 30), 2),
    "3d-div-divchan": (True, "default", None, ins(DIV_ONLY, normalizeInputChan="div"), (6, 10, 14), 2),
    "3d-all-unnormalized": (True, "default", None, ins(ALL, normalizeInput=False), (6, 10, 14), 1),
    "3d-n2-concat-all-skip": (True, "default", banks(2, "concat"), ins(ALL, addPressureSkip=True), (6, 10, 58), 2),
    "3d-n3-add-U": (True, "default", banks(3, "add"), ins(U_ONLY), (8, 20, 124), 2),
    "3d-n2-add-div-skip": (True, "default", banks(2, "add"), ins(DIV_ONLY, normalizeInputChan="div",
                                                               addPressureSkip=True), (4, 14, 60), 1),
    "3d-n3-concat-pU-skip": (True, "default", banks(3, "concat"), ins(P_U, addPressureSkip=True), (8, 12, 16), 2),
}


def run_forward(case, mode):
    orc = oracle.Oracle()
    is3d, model_type, bk, inputs, shape, nb = case
    batch = plume_batch(shape, is3d, nb=nb)
    mnp = synth.make_model(is3d, model_type=model_type, banks=bk, inputs=inputs)
    p0, inp = inputs_of(batch)
    wp, wU, wscale = oracle.model_forward(orc, mnp, p0, batch["UDiv"], batch["flags"])
    gm = fmodel.ProjectionModel.from_model(mnp)
    if mode != "default":
        gm.set_mode(mode)
    tol = MODE_TOL[gm.get_mode()]
    gp, gU = gm.forward(inp, return_scale=True)
    gp, gU = gp.cpu().numpy(), gU.cpu().numpy()
    for b in range(nb):
        assert abs(gm.last_scale[b] - wscale[b]) <= 1e-6 * wscale[b], (b, gm.last_scale, wscale)
        close(gp[b], wp[b], tol, "p[%d]" % b)
        close(gU[b], wU[b], tol, "U[%d]" % b)
    assert np.array_equal(gU == 0, wU == 0)
    return gm


@pytest.mark.parametrize("case", list(FP32))
def test_forward_fp32_graphs(case):
    gm = run_forward(FP32[case], "default")
    assert gm.get_mode() == "fp32"


@pytest.mark.parametrize("mode", ["default", "fp32", "tf32"])
@pytest.mark.parametrize("case", list(TC))
def test_forward_tensor_core_graph(case, mode):
    gm = run_forward(TC[case], mode)
    if mode == "default":
        assert gm.get_mode() == "tf32x3", "the 3-D 'default' graph stays on the tensor cores with any input block"


@pytest.mark.parametrize("chan", ["UDiv", "pDiv", "div", None])
@pytest.mark.parametrize("func", ["std", "norm"])
def test_scale(func, chan):
    """scale_out against the oracle's per entry, for each function and field; normalizeInput off (chan None): 1."""
    orc = oracle.Oracle()
    batch = plume_batch((6, 8, 10), True, nb=2)
    inputs = ins(ALL, normalizeInputFunc=func, normalizeInputChan=chan or "UDiv", normalizeInput=chan is not None)
    mnp = synth.make_model(True, inputs=inputs)
    p0, inp = inputs_of(batch)
    _, _, want = oracle.model_forward(orc, mnp, p0, batch["UDiv"], batch["flags"])
    for mode in ("tf32x3", "fp32"):
        gm = fmodel.ProjectionModel.from_model(mnp)
        gm.set_mode(mode)
        gm.forward(inp, return_scale=True)
        if chan is None:
            assert np.all(gm.last_scale == np.float32(1.0))
        else:
            assert np.all(np.abs(gm.last_scale - want) <= 1e-6 * want), (gm.last_scale, want)


# The six creators, with the arguments between ksize and weights: all NULL or 0 (the single-bank graph, the default
# input block, no normalization).
CREATORS = {"tfl_cnn_create": [], "tfl_cnn_create_graph": [None, None, 0, 0],
            "tfl_cnn_create_banked": [None, None, 0, 0, None],
            "tfl_cnn_create_model": [None, None, 0, 0, None, None],
            "tfl_cnn_create_model_ex": [None, None, 0, 0, None, None],
            "tfl_cnn_create_model_norm": [None, None, 0, 0, None, None, None]}


def create_via(gm, creator, mnp, cin="layers"):
    """(rc, handle) of `creator` on mnp's single-bank layers in gm's context; cin: a list, None (NULL), or the
    layers' input channels."""
    layers = mnp["layers"]
    n = len(layers)
    arr = lambda v: (C.c_int32 * n)(*v)
    cin = [w.shape[1] for w, _ in layers] if cin == "layers" else cin
    wp = (C.POINTER(C.c_float) * n)(*[w.ctypes.data_as(C.POINTER(C.c_float)) for w, _ in layers])
    bp = (C.POINTER(C.c_float) * n)(*[b.ctypes.data_as(C.POINTER(C.c_float)) for _, b in layers])
    h = C.c_void_p()
    rc = getattr(gm.ctx.lib, creator)(gm.ctx.h, 1 if mnp["is3D"] else 0, n, None if cin is None else arr(cin),
                                      arr([w.shape[0] for w, _ in layers]), arr([w.shape[4] for w, _ in layers]),
                                      *CREATORS[creator], wp, bp, C.byref(h))
    return rc, h


def twin(mnp, creator):
    """The model `creator` builds for mnp's single-bank layers, in a ProjectionModel shell."""
    gm = fmodel.ProjectionModel.from_model(mnp)
    rc, h = create_via(gm, creator, mnp)
    gm.ctx.check(rc)
    gm.ctx.lib.tfl_cnn_destroy(gm.ctx.h, gm.h)
    gm.h = h
    return gm


@pytest.mark.parametrize("is3d", [True, False], ids=["3d", "2d"])
def test_default_block_is_the_banked_model(is3d):
    """Every creator builds the model of tfl_cnn_create_model with the default block: the same bits in every mode.
    Each refuses a channel mismatch with the same message, and a NULL cin as a bad argument."""
    shape = (8, 12, 16) if is3d else (1, 24, 20)
    batch = plume_batch(shape, is3d, nb=2)
    mnp = synth.make_model(is3d, inputs=ins())
    _, inp = inputs_of(batch)
    a = fmodel.ProjectionModel.from_model(mnp)
    cin = [w.shape[1] for w, _ in mnp["layers"]]
    cin[2] += 1
    for creator in CREATORS:
        b = twin(mnp, creator)
        for mode in (["tf32x3", "tf32", "fp32"] if is3d else ["fp32"]):
            a.set_mode(mode)
            b.set_mode(mode)
            for x, y in zip(a.forward(inp), b.forward(inp)):
                assert torch.equal(x.view(torch.int32), y.view(torch.int32)), (creator, mode)
        for bad, msg in ((cin, "cnn: channel mismatch at layer 2"), (None, "cnn: bad arguments")):
            rc, h = create_via(a, creator, mnp, cin=bad)
            assert rc != 0 and not h.value, creator
            assert a.ctx.lib.tfl_last_error(a.ctx.h).decode() == msg, creator


@pytest.mark.parametrize("split", [1, 0], ids=["tf32x3", "tf32"])
@pytest.mark.parametrize("in_ch", [4, 5, 6])
def test_layer1_with_udiv_on_two_planes(in_ch, split):
    """Layer 1 of a set with UDiv: the two-plane kernel with 8-channel weights zero past the model's channels."""
    x, w, b, _ = make_layer("scaled", 8, False, (7, 9, 31), 2, seed=100 + in_ch)
    x[:, in_ch:] = 0.0
    w[:, in_ch:] = 0.0
    check_layer("l1-udiv-%d" % in_ch, x, w, b, None, split)


def _hooks():
    from fluidnet_b200 import _lib
    lib = _lib.load()
    P = C.c_void_p
    lib.tfl_debug_tc_pyramid2.argtypes = [P, P, P] + [C.c_int] * 8
    lib.tfl_debug_cnn_inputs_padded.argtypes = [P] * 7 + [C.c_int] * 4
    return lib


@pytest.mark.parametrize("ch", [ALL, U_ONLY, P_U, DIV_ONLY, dict(pDiv=True, UDiv=False, div=True, flags=True)],
                         ids=["all", "U", "pU", "div", "default"])
def test_padded_input_is_the_oracle_input(ch):
    """The tensor-core input planes hold the oracle's scaled channels bit for bit (same scale), zero past them; a
    set without UDiv leaves the second plane alone."""
    from fluidnet_b200 import tfluids
    orc = oracle.Oracle()
    nb, shape = 2, (6, 9, 13)
    batch = plume_batch(shape, True, nb=nb)
    p0, _ = inputs_of(batch)
    x, _, _, _, scales = model_input(orc, {"inputs": ins(ch)}, p0, batch["UDiv"], batch["flags"])
    U1 = batch["UDiv"].copy()
    orc.setWallBcsForward(U1, batch["flags"], as_mask_multiply=True)
    gm = fmodel.ProjectionModel.from_model(synth.make_model(True, inputs=ins(ch)))
    px, py = layout(nb, *shape)
    out = torch.full((nb, 2, shape[0] + 2, py, px, 4), float(SENTINEL), device="cuda")
    dev = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (p0, U1, batch["flags"])]
    ctx = tfluids._ctx_for(dev[0])
    ctx.check(_hooks().tfl_debug_cnn_inputs_padded(ctx.h, gm.h, *[d.data_ptr() for d in dev],
                                                   scales.ctypes.data, out.data_ptr(), nb, *shape))
    got = out.cpu().numpy()
    c = x.shape[1]
    inner = unpack(got, *shape)
    assert np.array_equal(inner[:, :c].view(np.uint32), x.view(np.uint32))
    if ch["UDiv"]:
        assert np.all(inner[:, c:] == 0.0)
    else:
        assert np.all(inner[:, c:4] == 0.0) and is_sentinel(got[:, 1]).all()


@pytest.mark.parametrize("phase", [0, 1])
def test_two_plane_pyramid_on_a_plane_range(phase):
    """Both float4 planes pooled, all four channels each, in k_pool's order (bit for bit); other output planes keep
    their bits."""
    from fluidnet_b200 import tfluids
    nb, nz_in, ny, nx = 2, 13, 6, 10
    nz_out, z_lo, z_hi = 6, 1, 5
    rs = np.random.RandomState(17 + phase)
    x = rs.uniform(-1, 1, (nb, 8, nz_in, ny, nx)).astype(np.float32)
    px, py = layout(nb, nz_in, ny, nx)
    hin = pack(x, px, py)
    used = np.zeros(nz_in, bool)
    used[2 * z_lo + phase:2 * z_hi + phase] = True
    hin[:, :, 1:nz_in + 1][:, :, ~used] = np.nan
    qx, qy = layout(nb, nz_out, ny // 2, nx // 2)
    hout = np.full((nb, 2, nz_out + 2, qy, qx, 4), SENTINEL, np.float32)
    din, dout = torch.from_numpy(hin).cuda(), torch.from_numpy(hout).cuda()
    ctx = tfluids._ctx_for(din)
    ctx.check(_hooks().tfl_debug_tc_pyramid2(ctx.h, din.data_ptr(), dout.data_ptr(), nb, nz_in, ny, nx, nz_out, phase,
                                             z_lo, z_hi))
    got = dout.cpu().numpy()
    want = hout.copy()
    for z in range(z_lo, z_hi):
        acc = np.zeros((nb, 8, ny // 2, nx // 2), np.float32)
        for dz in range(2):
            for dy in range(2):
                for dx in range(2):
                    acc = (acc + x[:, :, 2 * z + phase + dz, dy::2, dx::2]).astype(np.float32)
        acc = (acc / np.float32(8.0)).reshape(nb, 2, 4, ny // 2, nx // 2).transpose(0, 1, 3, 4, 2)
        want[:, :, z + 1, 1:ny // 2 + 1, 1:nx // 2 + 1, :] = acc
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


def test_step_and_its_graph():
    """One tfl_simulate_step with a UDiv + skip model (the per-operator path) against oracle.simulate, and the step
    graph replaying it bit for bit."""
    from fluidnet_b200 import simulate
    orc = oracle.Oracle()
    n = 24
    batch = plume_batch((n, n, n), True, inflow=n / 128.0 * 4)
    mnp = synth.make_model(True, inputs=ins(ALL, addPressureSkip=True))
    gm = fmodel.ProjectionModel.from_model(mnp)
    assert gm.get_mode() == "tf32x3"
    mconf = step_mconf(n)
    ga = to_gpu(batch)
    gb = to_gpu(batch)
    simulate.simulate_fused(None, mconf, ga, gm)
    oracle.simulate(orc, mconf, batch, mnp)
    for k in ("density", "UDiv", "pDiv"):
        close(ga[k].cpu().numpy(), batch[k], 2e-5, "step vs oracle " + k)
    stream = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(stream):
        simulate.simulate_fused(None, mconf, gb, gm)      # gb and ga now hold the same state
        graph = simulate.StepGraph(mconf, gb, gm)
        for _ in range(2):
            simulate.simulate_fused(None, mconf, ga, gm)
            graph.launch()
        stream.synchronize()
        for k in ("density", "UDiv", "pDiv"):
            assert torch.equal(ga[k].view(torch.int32), gb[k].view(torch.int32)), k
        graph.close()


def test_slab_refuses_a_non_default_block():
    from fluidnet_b200 import simulate, tfluids
    from fluidnet_b200.slab import NativeSlabSimulator
    dev = torch.device("cuda", 0)
    tb, mconf, _ = banked_problem(32, 16, 16, None)
    single = synth.make_model(True)
    sim = NativeSlabSimulator(tb, mconf, single["layers"], dev, rank=0, world=1)
    ctx, mc = sim.ctx, simulate.make_mconf(mconf)
    for inputs in (ins(ALL), ins(normalizeInputFunc="norm"), ins(addPressureSkip=True)):
        m = fmodel.ProjectionModel.from_model(synth.make_model(True, inputs=inputs))
        assert b"input block" in refused(ctx, lambda: ctx.lib.tfl_slab_sim_step(ctx.h, sim.h, C.byref(mc), m.h))
        g = torch.zeros(1, 1, 16, 16, 16, device=dev)
        u = torch.zeros(1, 3, 16, 16, 16, device=dev)
        sums = torch.zeros(2, dtype=torch.float64, device=dev)
        msg = refused(ctx, lambda: ctx.lib.tfl_cnn_project_from_sums(
            ctx.h, m.h, tfluids._grid(g), tfluids._grid(u), tfluids._grid(g), C.c_void_p(sums.data_ptr()),
            tfluids._grid(g), tfluids._grid(u), C.c_float(1e-5)))
        assert b"input block" in msg
    sim.close()


def test_unbuildable_blocks_are_refused():
    from fluidnet_b200._lib import TflError
    layers = synth.make_model(True)["layers"]
    for kw, msg in ((ins(dict(pDiv=False, UDiv=False, div=False, flags=True)), "any \\(U, div or p\\)"),
                    (ins(dict(pDiv=True, UDiv=False, div=False, flags=True)), "VelocityUpdate"),
                    (ins(U_ONLY, normalizeInputChan="div"), "'div' needs inputChannels.div"),
                    (ins(ALL), "first layer takes 3"),                       # cin[0] of the default set
                    (ins(addPressureSkip=True), "cout\\[3\\] \\+ 1")):       # the last layer lacks pDiv's channel
        with pytest.raises(TflError, match=msg):
            fmodel.ProjectionModel(layers, True, **kw)
    yang = synth.make_model(True, model_type="yang", inputs=ins(ALL))
    with pytest.raises(TflError, match="yang model must not have UDiv"):
        fmodel.ProjectionModel.from_model(yang)
    tog = synth.make_model(True, model_type="tog")
    with pytest.raises(TflError, match="addPressureSkip"):
        fmodel.ProjectionModel(tog["layers"], True, pool=tog["pool"], up=tog["up"], addPressureSkip=True)
