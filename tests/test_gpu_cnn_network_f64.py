"""The whole projection network (tfl_cnn_project: the input block, the graph driver between kernels, the skip and the
finish) against float64 with the per-voxel bound of tests/network_bound.py, on every path the library dispatches:
|GPU - float64| <= E at every voxel of p and U, the worst voxel and its err / E in the message.

Every case asserts the mode the model takes at creation (3xTF32 where the tensor cores cover the graph,
network_bound.tc_covered, else fp32); graphs the tensor cores do not cover run in fp32 only, and
test_tensor_core_modes_refused checks that set_mode refuses the tensor-core modes for them.  On the tensor cores each
case is labelled with the convolution kernel the host's predicate picks (nx <= 128 the z-streaming kernel, wider rows
the box kernel, restated as in test_gpu_conv_tc_zstream.py; nothing observes the launch itself).  The GPU's scale
(return_scale) must lie in network_bound.scale_interval.

The fused step (tfl_simulate_step, 64^3 and 128^3 in 3xTF32, direct and as a replayed step graph) and the emulated
z-slabs (world 2 and 3 on one GPU) do not return their scale: they are checked on the scale interval
(forward_bound(scale=None)), against the float64 projection of the pre-projection state.  That state comes from the
operator sequence (simulate.simulate(outputDiv=True) and setConstVals), which the step tests pin bit-exact; the
U BCs and the +-1e6 clamp that follow the projection are applied to the float64 result as well.

Inputs: the smooth plume velocity, the uniform-random +-2 field, and exotic flags (obstacles, Empty and Outflow
cells, where the pressure is small and the finish takes its other branches).  Non-vacuity: the TF32 output at 64^3
fails the 3xTF32 bound.

Largest err / E measured on an H100 80GB HBM3 (SXM, 700 W power limit) over all cases, p / U (each case prints its
own):
  fp32 0.14 / 0.46;
  3xTF32 0.063 / 0.46;
  TF32 0.043 / 0.46;
  fused step and graph replay 0.063 / 0.20;
  z-slabs 0.014 / 0.21;
  TF32 against the 3xTF32 bound 1.89 / 1.17.
U's ratio is the finish's own rounding.  p's ratios are small because sum |w| E assumes every error lines up, which
signed weights do not do (DESIGN.md section 1).  The float64 side takes about 10 s of CPU at 128^3 and about
a minute for the file."""
import os

import numpy as np
import pytest
import torch

import oracle
from fluidnet_b200 import synth
from fluidnet_b200._lib import TflError
from network_bound import check, excess, forward_bound, tc_covered
from test_gpu_cnn_bn import make_gpu

pytestmark = pytest.mark.gpu

WW_MAX = 128            # widest row of the z-streaming tensor-core kernel (k_conv3_tc_z)
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "myModel2D_layers.npz")


def banks(num, agg, kind="mres", s=1, j=3):
    return {"num": num, "split_stage": s, "join_stage": j, "aggregate": agg, "type": kind}


def make_inputs(shape, is3d, nb, kind, seed=11):
    """(pDiv, UDiv, flags): 'plume' smooth velocity, 'random' uniform +-2, 'exotic' random on exotic flags."""
    nz, ny, nx = shape
    flags = synth.make_flags(nx, ny, nz, is3d, nb=nb, geometry=True, exotic=kind == "exotic", seed=seed)
    if kind == "plume":
        U = synth.make_smooth_velocity(flags, is3d, amp=3.0, seed=seed)
    else:
        U = synth.make_velocity(flags, is3d, amp=2.0, seed=seed)
    oracle.Oracle().setWallBcsForward(U, flags)
    rs = np.random.RandomState(seed + 1)
    pDiv = ((rs.rand(*flags.shape) - 0.5) * 0.2).astype(np.float32)
    return pDiv, np.ascontiguousarray(U, np.float32), np.ascontiguousarray(flags)


def kernel_path(model, mode, nx):
    if mode == "fp32":
        return "fp32"
    return "%s %s" % (mode, "zstream" if nx <= WW_MAX else "box")


def run_case(what, model, shape, nb, mode, kind="plume"):
    """Forward on the GPU in `mode` and the per-voxel check.  Returns max err / E over p and U."""
    pDiv, U, flags = make_inputs(shape, model["is3D"], nb, kind)
    gm = make_gpu(model)
    assert gm.get_mode() == ("tf32x3" if tc_covered(model) else "fp32"), (what, gm.get_mode())
    gm.set_mode(mode)
    gp, gU = gm.forward(tuple(torch.from_numpy(a).cuda() for a in (pDiv, U, flags)), return_scale=True)
    gp, gU = gp.cpu().numpy(), gU.cpu().numpy()
    ref = forward_bound(oracle.Oracle(), model, pDiv, U, flags, mode, scale=gm.last_scale)
    s = gm.last_scale.astype(np.float64)
    assert ((ref["s_lo"] <= s) & (s <= ref["s_hi"])).all(), (what, s, ref["s_lo"], ref["s_hi"])
    path = kernel_path(model, mode, shape[2])
    rp = check("%s [%s] p" % (what, path), gp, ref["p"], ref["Ep"])
    rU = check("%s [%s] U" % (what, path), gU, ref["U"], ref["EU"])
    print("network f64 %s [%s]: max err/E p %.3g U %.3g" % (what, path, rp, rU))
    return max(rp, rU)


def mode_params(table, model_of):
    """(case, mode) for every case of `table` in every mode its graph runs in: all three where the tensor cores
    cover it, fp32 otherwise."""
    out = []
    for case in table:
        modes = MODES if tc_covered(model_of(case)) else ["fp32"]
        out += [pytest.param(case, m, id="%s-%s" % (case, m)) for m in modes]
    return out


MODES = ["fp32", "tf32x3", "tf32"]

# 3-D 'default': the bench's 128^3 (nb = 1, plume), 64^3 nb = 2, tile-edge grids nb = 3, and rows on both sides of
# the z-streaming kernel's limit.
DEFAULT = {"128-nb1-plume": ((128, 128, 128), 1, "plume"), "64-nb2-random": ((64, 64, 64), 2, "random"),
           "7x9x31-nb3-exotic": ((7, 9, 31), 3, "exotic"), "13x17x61-nb3-random": ((13, 17, 61), 3, "random"),
           "nx128-exotic": ((6, 10, 128), 1, "exotic"), "nx129-random": ((6, 10, 129), 1, "random")}


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", list(DEFAULT))
def test_default_3d(case, mode):
    shape, nb, kind = DEFAULT[case]
    run_case("3d-default " + case, synth.make_model(True), shape, nb, mode, kind)


# Banks: 'mres' 2 and 3 banks concat / add (tensor cores: split 1 / join 3; a later split runs on fp32), 'dilate' on
# grids 2 and 4 do not divide.
BANKED = {
    "mres-n2-concat": (banks(2, "concat"), (8, 12, 20), 2, "random"),
    "mres-n3-add": (banks(3, "add"), (8, 12, 24), 2, "exotic"),
    "mres-n3-concat": (banks(3, "concat"), (8, 20, 36), 1, "plume"),
    "mres-n2-add-s2j4": (banks(2, "add", "mres", 2, 4), (6, 10, 12), 2, "random"),
    "dilate-n2-concat": (banks(2, "concat", "dilate"), (7, 10, 29), 2, "random"),
    "dilate-n3-add": (banks(3, "add", "dilate"), (9, 11, 13), 1, "exotic"),
}


@pytest.mark.parametrize("case,mode", mode_params(BANKED, lambda c: synth.make_model(True, banks=BANKED[c][0])))
def test_banks(case, mode):
    bk, shape, nb, kind = BANKED[case]
    run_case("3d " + case, synth.make_model(True, banks=bk), shape, nb, mode, kind)


def bn_model(train, bk=None, relu6=False):
    m = synth.make_model(True, banks=bk, batch_norm=None if train is None else {"train": train})
    if relu6:
        m["nonlinType"] = "relu6"
        first = m["layers"][0] if not isinstance(m["layers"][0], list) else m["layers"][0][0]
        first[0][...] *= np.float32(30.0)          # the first stage's values cross 6
    return m


# BN with running and batch statistics: single-bank on the tensor cores (and fp32), banked on fp32; relu6 banked on
# the tensor cores.
NORM = {
    "bn-batch": (lambda: bn_model(True), (8, 10, 12), 2),
    "bn-running": (lambda: bn_model(False), (8, 10, 12), 2),
    "bn-batch-relu6": (lambda: bn_model(True, relu6=True), (6, 9, 130), 1),
    "bn-running-relu6": (lambda: bn_model(False, relu6=True), (7, 9, 31), 2),
    "bn-batch-mres-n2-concat": (lambda: bn_model(True, banks(2, "concat")), (8, 12, 16), 2),
    "bn-running-dilate-n2-add": (lambda: bn_model(False, banks(2, "add", "dilate")), (7, 10, 13), 2),
    "relu6-mres-n2-concat": (lambda: bn_model(None, banks(2, "concat"), relu6=True), (8, 12, 16), 2),
    "relu6-dilate-n3-add": (lambda: bn_model(None, banks(3, "add", "dilate"), relu6=True), (7, 9, 11), 1),
}


@pytest.mark.parametrize("case,mode", mode_params(NORM, lambda c: NORM[c][0]()))
def test_bn_and_relu6(case, mode):
    make, shape, nb = NORM[case]
    run_case("3d " + case, make(), shape, nb, mode, "random")


# The input block: channel sets, 'norm', the normalisation channel, the skip, normalizeInput = false.
INPUTS = {
    "all-channels": {"inputChannels": {"UDiv": True}},
    "udiv-only": {"inputChannels": {"pDiv": False, "UDiv": True, "div": False}},
    "norm": {"normalizeInputFunc": "norm"},
    "chan-pdiv": {"normalizeInputChan": "pDiv"},
    "chan-div": {"normalizeInputChan": "div"},
    "skip": {"addPressureSkip": True},
    "skip-udiv-norm": {"addPressureSkip": True, "inputChannels": {"UDiv": True}, "normalizeInputFunc": "norm"},
    "no-normalize": {"normalizeInput": False},
}


@pytest.mark.parametrize("case,mode", mode_params(INPUTS, lambda c: synth.make_model(True, inputs=INPUTS[c])))
def test_input_block(case, mode):
    run_case("3d inputs " + case, synth.make_model(True, inputs=INPUTS[case]), (7, 10, 21), 2, mode, "exotic")


OTHER = {
    "3d-tog": (lambda: synth.make_model(True, model_type="tog"), (16, 16, 24), 2, "random"),
    "3d-yang": (lambda: synth.make_model(True, model_type="yang"), (6, 8, 10), 2, "exotic"),
    "2d-tog": (lambda: synth.make_model(False, model_type="tog"), (1, 32, 48), 2, "exotic"),
    "2d-default": (lambda: synth.make_model(False), (1, 36, 51), 2, "random"),
    "2d-tog-max-pool": (lambda: dict(synth.make_model(False, model_type="tog"), poolType="max"), (1, 32, 48), 1,
                        "random"),
}


@pytest.mark.parametrize("case", list(OTHER))
def test_other_graphs(case):
    make, shape, nb, kind = OTHER[case]
    run_case(case, make(), shape, nb, "fp32", kind)


@pytest.mark.parametrize("n", [64, 128])
def test_my_model_2d(n):
    z = np.load(GOLD)
    layers = [(np.ascontiguousarray(z["w%d" % l], np.float32), np.ascontiguousarray(z["b%d" % l], np.float32))
              for l in range(int(z["n_layers"]))]
    run_case("myModel2D %d^2" % n, {"is3D": False, "layers": layers}, (1, n, n), 1, "fp32", "plume")


def test_tf32_fails_the_3xtf32_bound():
    """Non-vacuity: the TF32 mode's output at 64^3 on the signed random field exceeds the 3xTF32 bound."""
    model = synth.make_model(True)
    pDiv, U, flags = make_inputs((64, 64, 64), True, 1, "random")
    gm = make_gpu(model)
    gm.set_mode("tf32")
    gp, gU = gm.forward(tuple(torch.from_numpy(a).cuda() for a in (pDiv, U, flags)), return_scale=True)
    ref = forward_bound(oracle.Oracle(), model, pDiv, U, flags, "tf32x3", scale=gm.last_scale)
    rp = excess(gp.cpu().numpy(), ref["p"], ref["Ep"])[0]
    rU = excess(gU.cpu().numpy(), ref["U"], ref["EU"])[0]
    print("network f64 tf32 against the 3xTF32 bound: max err/E p %.3g U %.3g" % (rp, rU))
    assert max(rp, rU) > 1.0, "TF32 stays within the 3xTF32 bound (p %.3g, U %.3g): the bound has no teeth" % (rp, rU)


UNCOVERED = {**{"3d " + c: (lambda c=c: synth.make_model(True, banks=BANKED[c][0])) for c in BANKED},
             **{"3d " + c: NORM[c][0] for c in NORM}, **{c: OTHER[c][0] for c in OTHER}}
UNCOVERED = {c: make for c, make in UNCOVERED.items() if not tc_covered(make())}


@pytest.mark.parametrize("case", list(UNCOVERED))
def test_tensor_core_modes_refused(case):
    """The graphs the cases above run in fp32 only: the model starts in fp32 and set_mode refuses both tensor-core
    modes."""
    gm = make_gpu(UNCOVERED[case]())
    assert gm.get_mode() == "fp32"
    for mode in ("tf32x3", "tf32"):
        with pytest.raises(TflError):
            gm.set_mode(mode)
        assert gm.get_mode() == "fp32"


# ---------------------------------------------------------------------------------------------------------------
# The fused step and the z-slabs: the scale interval
# ---------------------------------------------------------------------------------------------------------------
def step_problem(n, seed=21):
    """A plume problem at n^3 with a small signed pDiv (the network's pDiv channel), and its mconf."""
    flags = synth.make_flags(n, n, n, True, nb=1, geometry=True)
    U = synth.make_smooth_velocity(flags, True, amp=3.0, seed=seed)
    oracle.Oracle().setWallBcsForward(U, flags)
    pDiv = ((np.random.RandomState(seed).rand(*flags.shape) - 0.5) * 0.2).astype(np.float32)
    batch = {"pDiv": pDiv, "UDiv": U, "flags": flags, "density": synth.make_density(flags)}
    oracle.create_plume_bcs(batch, [1.0], n / 128.0 * 4, 0.15)
    mconf = oracle.default_mconf(dt=0.1, maccormackStrength=0.6, buoyancyScale=2.0 * n / 128,
                                 vorticityConfinementAmp=3.0, simMethod="convnet")
    return batch, mconf


def projection_reference(state, mconf, gm, mnp):
    """The float64 projection of one step from `state` (GPU tensors, left as they are) on the scale interval: the
    operator sequence up to the projection and setConstVals, forward_bound, then the U BCs (x inv + bc: E |inv| plus
    two roundings) and the +-1e6 clamp (1-Lipschitz)."""
    from fluidnet_b200 import simulate
    from network_bound import gamma
    ob = {k: v.clone() for k, v in state.items()}
    simulate.simulate(None, mconf, ob, gm, outputDiv=True)
    p, U, flags, density = simulate.getPUFlagsDensityReference(ob)
    simulate.setConstVals(ob, p, U, flags, density)
    assert ob.get("pBC") is None, "a pressure BC takes the operator path, not these cases"
    ref = forward_bound(oracle.Oracle(), mnp, p.cpu().numpy(), U.cpu().numpy(), flags.cpu().numpy(), gm.get_mode(),
                        scale=None, threshold=gm.threshold)
    inv, bc = ob["UBCInvMask"].cpu().numpy().astype(np.float64), ob["UBC"].cpu().numpy().astype(np.float64)
    Ui = ref["U"] * inv
    ref["EU"] = ref["EU"] * np.abs(inv) + gamma(2) * (np.abs(Ui) + ref["EU"] * np.abs(inv) + np.abs(bc))
    ref["U"] = np.clip(Ui + bc, -1e6, 1e6)
    return ref


def check_step(what, p, U, ref):
    rp = check(what + " p", p.cpu().numpy(), ref["p"], ref["Ep"])
    rU = check(what + " U", U.cpu().numpy(), ref["U"], ref["EU"])
    print("network f64 %s: max err/E p %.3g U %.3g (scale interval rel. width %.2g)" % (
        what, rp, rU, float(((ref["s_hi"] - ref["s_lo"]) / ref["s_lo"]).max())))


@pytest.mark.parametrize("n", [64, 128])
def test_fused_step(n):
    """One tfl_simulate_step in 3xTF32 (the fused path: k_vort_bc_mask's statistics, k_cnn_inputs_fused, the
    tensor-core stack, k_cnn_finish_fused)."""
    from fluidnet_b200 import simulate
    from test_gpu_step_paths import takes_fused_path
    batch, mconf = step_problem(n)
    mnp = synth.make_model(True)
    gm = make_gpu(mnp)
    assert gm.get_mode() == "tf32x3" and takes_fused_path({"mode": gm.get_mode(), "nb": 1, "pbc": False})
    gb = {k: torch.from_numpy(v.copy()).cuda() for k, v in batch.items()}
    state = {k: v.clone() for k, v in gb.items()}
    simulate.simulate_fused(None, mconf, gb, gm)
    torch.cuda.synchronize()
    check_step("fused step %d^3 [tf32x3]" % n, gb["pDiv"], gb["UDiv"], projection_reference(state, mconf, gm, mnp))


def test_fused_step_graph_replay():
    """The same step replayed from a step graph (tfl_step_graph_launch), 64^3, after one direct step."""
    from fluidnet_b200 import simulate
    batch, mconf = step_problem(64, seed=23)
    mnp = synth.make_model(True)
    gm = make_gpu(mnp)
    g = {k: torch.from_numpy(v.copy()).cuda() for k, v in batch.items()}
    stream = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(stream):
        simulate.simulate_fused(None, mconf, g, gm)
        graph = simulate.StepGraph(mconf, g, gm)
        stream.synchronize()
        state = {k: v.clone() for k, v in g.items()}
        stream.synchronize()
        graph.launch()
        stream.synchronize()
        graph.close()
    torch.cuda.synchronize()
    check_step("step graph replay 64^3 [tf32x3]", g["pDiv"], g["UDiv"], projection_reference(state, mconf, gm, mnp))


@pytest.mark.parametrize("world", [2, 3])
def test_emulated_slabs(world):
    """One step of the z-slab driver with `world` slabs on one GPU (as test_gpu_slab.py::
    test_emulated_slabs_on_one_gpu): each rank's projection (tfl_cnn_project_from_sums on the all-reduced sums) within
    the bound on its owned planes."""
    from fluidnet_b200.slab import SlabSimulator, run_lockstep
    from test_gpu_slab import _problem
    batch, mconf, mnp = _problem(48)
    tb = {k: torch.from_numpy(v) for k, v in batch.items()}
    sims = [SlabSimulator(tb, mconf, mnp["layers"], torch.device("cuda", 0), rank=r, world=world)
            for r in range(world)]
    assert all(q.model.get_mode() == "tf32x3" for q in sims)
    state = {k: v.cuda() for k, v in tb.items()}
    run_lockstep(sims)
    torch.cuda.synchronize()
    got = {k: torch.cat([q.dec.owned(q.s[k]).cpu() for q in sims], dim=2) for k in ("pDiv", "UDiv")}
    assert sims[0].ctx.trace_faults() == 0
    check_step("z-slabs world %d 48^3 [tf32x3]" % world, got["pDiv"], got["UDiv"],
               projection_reference(state, mconf, sims[0].model, mnp))
