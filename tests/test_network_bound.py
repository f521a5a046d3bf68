"""CPU checks of the whole-network bound (tests/network_bound.py): it holds for a float32 emulation of the library's
arithmetic, it fails for that emulation with one fault injected, and the batch-statistics BN rule holds for perturbed
float64 inputs.

`F32` is oracle.model.F64's set of operations in float32 the way the fp32 kernels compute them: a convolution starts from
the bias and adds one fmaf per term in the order (c, dz, dy, dx) (one rounding per term: the float32 product is exact
in float64), average pooling sums in order and divides, BN rounds a and c once and applies a fused multiply-add, a
bank join 'add' sums in bank order.  The input block divides by the float32 scale, and the finish is the oracle's
float32 VelocityUpdate between the two scalings.  The faults, each of which must break the bound at some voxel:
  plane   one z-plane of layer 2's input taken from the neighbouring plane (a stale or shifted plane);
  bias    one output channel's bias dropped in layer 1;
  tf32    layer 3's operands truncated to TF32, checked against the 3xTF32 bound (a 3xTF32 layer without its lo terms);
  scale   entry 1 normalised (and scaled back) with entry 0's scale;
  pad     one non-zero cell in layer 1's zero padding, next to the obstacle border.
The faults run on the 3-D 'default' graph with the signed weights the GPU cases use and with non-negative weights
(nonneg_model).  plane, bias, scale and pad break the bound on both, by factors of 10 to 10^5.  tf32 breaks it on
non-negative weights only (err/E about 14): with signed weights the bound's sum |w| E has the slack of each layer's
cancellation, and TF32 truncation in layer 3 alone reaches only about 0.65 of it.  So the per-voxel check on signed
weights cannot see a single 3xTF32 layer that lost its lo terms; it does see the whole network in TF32 (the GPU
non-vacuity case, test_gpu_cnn_network_f64.py).  The whole file takes about 10 s of CPU."""
import numpy as np
import pytest

import oracle
from oracle.model import F64, batch_norm, network
from fluidnet_b200 import synth
from network_bound import (Bound, check, excess, forward_bound, input_fields, model_inputs, scale_intervals)
from scenes import bn_model

FAULTS = ("plane", "bias", "tf32", "scale", "pad")


def tf32(a):
    return (np.ascontiguousarray(a, np.float32).view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)


def f32_scale(field, kw, threshold=1e-5):
    """The GPU's scale in float32 (scale_from_sums without contraction) from float64 sums."""
    if not kw["normalizeInput"]:
        return np.float32(1.0)
    f = np.asarray(field, np.float32).ravel()
    s1, s2 = np.float32(f.astype(np.float64).sum()), np.float32((f * f).astype(np.float64).sum())
    if kw["normalizeInputFunc"] == "norm":
        return max(np.sqrt(s2), np.float32(threshold))
    n = f.size
    t = (s2 * np.float32(n) + np.float32(-1.0) * (s1 * s1)) / np.float32(float(n) * float(n - 1))
    return max(np.sqrt(t), np.float32(threshold))


class F32:
    """F64's operations in the float32 arithmetic of the fp32 kernels; `fault` injects one of FAULTS."""

    def __init__(self, fault=None):
        self.fault = fault

    lift = staticmethod(lambda x: np.asarray(x, np.float32))

    def conv(self, x, w, b, is3d, d, li, relu):
        x, w, b = np.asarray(x, np.float32), np.asarray(w, np.float32), np.asarray(b, np.float32).copy()
        if self.fault == "plane" and li == 1:
            x = x.copy()
            z = x.shape[2] // 2
            x[:, :, z] = x[:, :, z + 1]
        if self.fault == "bias" and li == 0:
            b[3] = 0.0
        if self.fault == "tf32" and li == 2:
            x, w = tf32(x), tf32(w)
        cout, cin, kz, k, _ = w.shape
        pz, p = d * (kz - 1) // 2, d * (k - 1) // 2
        B, _, Z, Y, X = x.shape
        xp = np.zeros((B, cin, Z + 2 * pz, Y + 2 * p, X + 2 * p), np.float32)
        xp[:, :, pz:pz + Z, p:p + Y, p:p + X] = x
        if self.fault == "pad" and li == 0:
            xp[0, cin - 1, pz + Z // 2, p + Y // 2, 0] = 1.0        # left of x = 0, an obstacle column
        acc = np.broadcast_to(b[None, :, None, None, None], (B, cout, Z, Y, X)).astype(np.float32)
        w64 = w.astype(np.float64)
        for c in range(cin):
            for tz in range(kz):
                for ty in range(k):
                    for tx in range(k):
                        sl = xp[:, c, tz * d:tz * d + Z, ty * d:ty * d + Y, tx * d:tx * d + X].astype(np.float64)
                        acc = (acc + w64[:, c, tz, ty, tx][None, :, None, None, None] * sl[:, None]).astype(np.float32)
        return self.nonlin(acc, "relu") if relu else acc

    shuffle = staticmethod(F64.shuffle)

    @staticmethod
    def nonlin(x, kind):
        if kind == "sigmoid":
            return (np.float32(1.0) / (np.float32(1.0) + np.exp(-x))).astype(np.float32)
        if kind == "relu6":
            return np.minimum(np.maximum(x, np.float32(0.0)), np.float32(6.0))
        return np.maximum(x, np.float32(0.0))

    @staticmethod
    def pool(x, q, is3d, kind):
        b_, c_, z_, y_, x_ = x.shape
        qz = q if is3d else 1
        v = x.reshape(b_, c_, z_ // qz, qz, y_ // q, q, x_ // q, q)
        if kind == "max":
            return v.max(axis=(3, 5, 7))
        acc = np.zeros((b_, c_, z_ // qz, y_ // q, x_ // q), np.float32)
        for dz in range(qz):
            for dy in range(q):
                for dx in range(q):
                    acc = acc + v[:, :, :, dz, :, dy, :, dx]
        return (acc / np.float32(qz * q * q)).astype(np.float32)

    @staticmethod
    def bn(x, e, train, li):
        c_ = x.shape[1]
        w = np.ones(c_) if e.get("weight") is None else np.asarray(e["weight"], np.float64)
        b = np.zeros(c_) if e.get("bias") is None else np.asarray(e["bias"], np.float64)
        eps = float(np.float32(e["eps"]))
        if train:
            x64 = x.astype(np.float64)
            mean = x64.mean(axis=(0, 2, 3, 4))
            var = x64.var(axis=(0, 2, 3, 4))
        else:
            mean, var = np.asarray(e["running_mean"], np.float64), np.asarray(e["running_var"], np.float64)
        a = w / np.sqrt(var + eps)
        c = b - mean * a
        s = lambda t: t.astype(np.float32).astype(np.float64)[None, :, None, None, None]
        return (s(a) * x.astype(np.float64) + s(c)).astype(np.float32)

    up = staticmethod(F64.up)
    concat = staticmethod(F64.concat)

    @staticmethod
    def add(hs):
        acc = hs[0]
        for h in hs[1:]:
            acc = (acc + h).astype(np.float32)
        return acc


def emulate(be, model, pDiv, UDiv, flags, fault=None):
    """The library's forward in float32 (F32), with one fault.  Returns (p, U, scales)."""
    kw = model_inputs(model)
    fields = input_fields(be, pDiv, UDiv, flags)
    field = fields[{"UDiv": "U1", "pDiv": "pDiv", "div": "div"}[kw["normalizeInputChan"]]]
    B = flags.shape[0]
    scales = np.array([f32_scale(field[b], kw) for b in range(B)], np.float32)
    used = scales.copy()
    if fault == "scale":
        used[1] = used[0]
    sc = used.reshape(B, 1, 1, 1, 1)
    ch = dict({"pDiv": True, "UDiv": False, "div": True}, **(kw["inputChannels"] or {}))
    xs = [(fields[k] / sc).astype(np.float32) for k, on in (("pDiv", ch["pDiv"]), ("U1", ch["UDiv"]), ("div", ch["div"]))
          if on]
    x0 = np.concatenate(xs + [fields["occ"]], axis=1)
    ops = F32(fault)
    if kw["addPressureSkip"]:
        w, b = model["layers"][-1]
        h = network(model, x0, ops, hidden=True)
        body = ops.conv(h, w[:, :-1], b, model["is3D"], 1, len(model["layers"]) - 1, False)
        pS = (fields["pDiv"] / sc).astype(np.float32)
        pn = (body + (np.float32(w[0, -1].ravel()[0]) * pS).astype(np.float32)).astype(np.float32)
    else:
        pn = network(model, x0, ops)
    U = np.ascontiguousarray((fields["U1"] / sc).astype(np.float32))
    be.velocityUpdateForward(U, flags, pn)
    U = np.ascontiguousarray((U * sc).astype(np.float32))
    be.setWallBcsForward(U, flags, as_mask_multiply=True)
    return (pn * sc).astype(np.float32), U, scales


def problem(shape, is3d, nb, exotic=True, seed=5):
    """Flags with obstacles (and Empty / Outflow cells), a signed random velocity per entry at its own amplitude, and
    a small signed pDiv."""
    nz, ny, nx = shape
    flags = synth.make_flags(nx, ny, nz, is3d, nb=nb, geometry=True, exotic=exotic)
    rs = np.random.RandomState(seed)
    U = synth.make_velocity(flags, is3d, amp=2.0, seed=seed) * np.arange(1, nb + 1, dtype=np.float32).reshape(-1, 1, 1, 1, 1)
    pDiv = (rs.rand(*flags.shape).astype(np.float32) - np.float32(0.5)) * np.float32(0.2)
    return pDiv, np.ascontiguousarray(U, np.float32), flags


SOUND = {
    "3d-default": (lambda: synth.make_model(True), (6, 9, 11), True, 2),
    "3d-mres-n2-concat": (lambda: synth.make_model(True, banks={"num": 2, "split_stage": 1, "join_stage": 3,
                                                                "aggregate": "concat"}), (8, 10, 12), True, 2),
    "3d-dilate-n2-add": (lambda: synth.make_model(True, banks={"num": 2, "split_stage": 1, "join_stage": 3,
                                                               "aggregate": "add", "type": "dilate"}), (7, 9, 11), True, 1),
    "3d-bn-batch": (lambda: bn_model(True), (6, 8, 10), True, 2),
    "3d-bn-running-skip": (lambda: bn_model(False, inputs={"addPressureSkip": True}), (6, 8, 10), True, 2),
    "3d-yang": (lambda: synth.make_model(True, model_type="yang"), (6, 8, 10), True, 1),
    "2d-tog": (lambda: synth.make_model(False, model_type="tog"), (1, 16, 24), False, 2),
    "2d-mres-n2-add-norm": (lambda: synth.make_model(False, banks={"num": 2, "split_stage": 1, "join_stage": 3,
                                                                   "aggregate": "add"},
                                                     inputs={"normalizeInputFunc": "norm",
                                                             "inputChannels": {"UDiv": True}}), (1, 20, 16), False, 2),
}


@pytest.fixture(scope="module")
def orc():
    return oracle.Oracle()


@pytest.mark.parametrize("case", list(SOUND))
def test_bound_holds_for_float32_emulation(orc, case):
    make, shape, is3d, nb = SOUND[case]
    model = make()
    pDiv, U, flags = problem(shape, is3d, nb)
    p, Ug, scales = emulate(orc, model, pDiv, U, flags)
    ref = forward_bound(orc, model, pDiv, U, flags, "fp32", scale=scales)
    assert ((ref["s_lo"] <= scales) & (scales <= ref["s_hi"])).all(), (scales, ref["s_lo"], ref["s_hi"])
    rp = check(case + " p", p, ref["p"], ref["Ep"])
    rU = check(case + " U", Ug, ref["U"], ref["EU"])
    # without the returned scale the bound widens by the interval: the emulation stays inside it
    wide = forward_bound(orc, model, pDiv, U, flags, "fp32")
    check(case + " p (scale interval)", p, wide["p"], wide["Ep"])
    check(case + " U (scale interval)", Ug, wide["U"], wide["EU"])
    print("%s: max err/E p %.3f U %.3f" % (case, rp, rU))


def nonneg_model():
    """The 3-D 'default' graph with |w| and |b|: nothing cancels past layer 1, so the bound is within a small factor
    of the rounding it allows (with signed weights it is looser by each layer's cancellation, sum |w| |x| / |sum w x|),
    and an error as systematic as TF32 truncation shows at full size."""
    m = synth.make_model(True)
    m["layers"] = [(np.abs(w), np.abs(b)) for w, b in m["layers"]]
    return m


FAULT_CASES = [("nonneg", f) for f in FAULTS] + [("signed", f) for f in FAULTS if f != "tf32"]


@pytest.mark.parametrize("weights,fault", FAULT_CASES, ids=["%s-%s" % c for c in FAULT_CASES])
def test_bound_catches_injected_fault(orc, weights, fault):
    model = nonneg_model() if weights == "nonneg" else synth.make_model(True)
    pDiv, U, flags = problem((6, 9, 11), True, 2)
    p, Ug, scales = emulate(orc, model, pDiv, U, flags, fault)
    mode = "tf32x3" if fault == "tf32" else "fp32"
    ref = forward_bound(orc, model, pDiv, U, flags, mode, scale=scales)
    rp = excess(p, ref["p"], ref["Ep"])[0]
    rU = excess(Ug, ref["U"], ref["EU"])[0]
    print("fault %s: max err/E p %.3g U %.3g" % (fault, rp, rU))
    assert max(rp, rU) > 1.0, "fault '%s' stays within the %s bound (p %.3g, U %.3g)" % (fault, mode, rp, rU)


def test_tf32_operands_stay_within_their_own_bound(orc):
    """The 'tf32' fault is the TF32 mode's arithmetic on layer 3: within the TF32 bound, so the fault above fails
    because the 3xTF32 bound is tighter, not because the emulation is broken."""
    model = synth.make_model(True)
    pDiv, U, flags = problem((6, 9, 11), True, 2)
    p, Ug, scales = emulate(orc, model, pDiv, U, flags, "tf32")
    ref = forward_bound(orc, model, pDiv, U, flags, "tf32", scale=scales)
    check("tf32 p", p, ref["p"], ref["Ep"])
    check("tf32 U", Ug, ref["U"], ref["EU"])


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_batch_statistics_rule(seed):
    """h' = h + r E with r in [-1, 1] (random, and at the signs +-1): BN with batch statistics of h' stays within
    the rule's bound of BN of h, in float64 (the float rounding terms only widen it)."""
    rs = np.random.RandomState(seed)
    c = 4
    h = rs.randn(2, c, 5, 6, 7) * np.array([1.0, 1e-2, 5.0, 1.0]).reshape(1, c, 1, 1, 1)
    h[:, 3] = np.maximum(h[:, 3], 0.0)
    E = rs.rand(*h.shape) * np.array([1e-3, 1e-4, 1e-2, 1e-6]).reshape(1, c, 1, 1, 1)
    e = {"weight": (0.5 + rs.rand(c)).astype(np.float32), "bias": (rs.rand(c) - 0.5).astype(np.float32),
         "running_mean": np.zeros(c, np.float32), "running_var": np.ones(c, np.float32), "eps": 1e-4}
    y, Ey = Bound(synth.make_model(True), "fp32").bn((h, E), e, True, 0)
    assert np.allclose(y, batch_norm(h, e, True), rtol=0, atol=0)
    worst = 0.0
    for r in (rs.uniform(-1, 1, h.shape), np.sign(rs.randn(*h.shape)), np.ones(h.shape), -np.ones(h.shape)):
        y2 = batch_norm(h + r * E, e, True)
        worst = max(worst, check("BN batch r", y2, y, Ey))
    print("batch-statistics BN: max err/E %.3f" % worst)


def test_scale_interval_contains_the_float32_scale(orc):
    for func, chan in (("std", "UDiv"), ("norm", "UDiv"), ("std", "pDiv"), ("std", "div")):
        model = synth.make_model(True, inputs={"normalizeInputFunc": func, "normalizeInputChan": chan})
        pDiv, U, flags = problem((6, 9, 11), True, 2)
        fields = input_fields(orc, pDiv, U, flags)
        lo, hi = scale_intervals(fields, model)
        kw = model_inputs(model)
        field = fields[{"UDiv": "U1", "pDiv": "pDiv", "div": "div"}[chan]]
        for b in range(2):
            s = f32_scale(field[b], kw)
            assert lo[b] <= s <= hi[b] and (hi[b] - lo[b]) <= 4e-6 * s, (func, chan, lo[b], s, hi[b])
