"""The whole projection network in float64 with a per-voxel bound on |GPU - float64|, for every path the library
dispatches: the fp32 kernels, the tensor cores in 3xTF32 and TF32, with or without BN, banks, relu6, sigmoid, pooling,
pixel shuffle, the input block and the pressure skip.

The network is oracle.model.network, run on (value, bound) pairs by `Bound`, whose operations mirror F64's; `E` is a
float64 array beside each float64 activation with |gpu - value| <= E at every voxel.  u = 2^-24 (float32),
gamma_n = n u / (1 - n u), S(m) = conv(m, |w|) + |b| with m >= |gpu input| (|x| + E), taken with the layer's dilation.

Rules, one per operation
  * Input block.  U1 (masked velocity), div and the occupancy come from the oracle and are bit-exact with the GPU
    (tests/test_gpu_operators.py).  x0 = v / s rounds once: E = u |x0| (0 for the occupancy).  Where the GPU returns s,
    the float64 network runs on that s.  The scale itself must lie in `scale_interval`: scale_from_sums
    (tfl_device.cuh) evaluated in float32 on the exact float64 sums, with each float conversion taken one float either
    side (the GPU's double sums run in another order) and the product-sum with and without contraction.  Where s is
    not returned (the fused step, z-slabs), the network runs on the interval's midpoint and the relative width
    rho = (s_hi - s_lo) / s_lo adds rho |x0|: |v / s_gpu - v / s_mid| <= |x0| |s_mid - s_gpu| / s_gpu.
  * Convolution.  E_out = kappa S(|x| + E_in) + conv(E_in, |w|): the exact convolution of the perturbed input
    moves by at most sum |w| E_in, and the kernel's rounding is within kappa of the sum of magnitudes.
      - fp32 path: one fmaf per term from the bias, n = cin taps + 1 terms, kappa = gamma_n
        (tests/test_gpu_conv_fp32.py).
      - tensor cores: the 3x3x3 layers kappa = KAPPA[mode] (2^-16 3xTF32, 2^-8 TF32; tests/test_gpu_conv_tc.py's
        derivation of the operand split and the fp32 accumulation); the 1x1x1 tail TAIL_ULPS = 2^-20 >= gamma_9 (eight
        fused multiply-adds and the join of the shuffle, as there).
  * ReLU, relu6: 1-Lipschitz, exact: E unchanged, except that where v + E <= 0 (relu6 also v - E >= 6) both results
    are the same clamp value and E = 0, and within E of the clamp E shrinks to the distance: clip(v + E, 0, E).  Sigmoid: 1/4-Lipschitz, plus SIGMOID_ULPS sigma for expf, the add
    and the divide (tests/test_gpu_conv_fp32.py).
  * Average pooling: a float sum in a fixed order and a divide, q^d roundings each within u of the sum of magnitudes:
    mean(E) + gamma_{q^d} mean(|v| + E).  Max pooling: |max a' - max a| <= max |a' - a|, so max(E).
  * Pixel shuffle and nearest up-sampling move values, so they move E.  Bank join 'concat' moves E; 'add' is a float
    sum in bank order (k_bank_join, or the staging of the tensor-core join): sum E + gamma_{N-1} sum (|v| + E).
  * BN, running statistics: a = w / sqrt(var + eps), c = b - mean a in double, each rounded once to float, then
    a x + c (fused or not): E = |a| E_in + gamma_3 (|a| (|x| + E_in) + |c|) (the epilogue of test_tc_bn_layer and the
    BN kernels of test_gpu_cnn_bn.py).  On the tensor cores BN3 and BN4 are folded into w4 / b4 and w5 / b5 at
    creation instead: w' = w a and b' = b + w c, each rounded once, so the BN passes E_in |a| on with no rounding and
    the next layer takes m = |a| (|x| + E_in) + |c| >= the folded operands' magnitudes, with kappa + 2u
    (u for w' and b', u for |w'| <= (1 + u) |w a|).
  * BN, batch statistics, over the N = batch x voxels values of a channel, the GPU's h' = h + delta, |delta| <= E:
      |d mean| <= mean(E)                       the mean is linear;
      |d sigma| <= rms(E)                       Minkowski on the centred vector: ||(h + delta) - mean(h + delta)|| -
                                                ||h - mean h|| <= ||delta - mean delta|| <= ||delta||;
      |d sd| <= |d sigma|                       sd = sqrt(sigma^2 + eps) is 1-Lipschitz in sigma;
      |d a| <= |w| |d sd| / (sd sd_lo)          a = w / sd, sd_lo = sqrt(max(sigma - |d sigma|, 0)^2 + eps) bounds
                                                sd' below;
    the fp64 sums add (N + 4) 2^-53 of the sums of magnitudes to mean and variance (the variance's share enters sd
    through |sqrt(p) - sqrt(q)| <= sqrt(|p - q|)).  Then y' - y = a' (delta - d mean) + (a' - a) (h - mean), and
    the finalize kernel's float roundings of a and c and the apply add gamma_3 (|a'| (|h| + E) + |c'|).
  * Pressure skip (k_cnn_skip): p_net + w_skip (pDiv / s), three roundings: gamma_3 (|p_body| + E_body + |w_skip pS|);
    on the scale interval also rho |w_skip pS|, as for x0.
  * Finish (k_cnn_finish / k_cnn_finish_fused, -fmad=false): U = setWallBcs((U1 / s - g) s) with g the pressure
    term of VelocityUpdate (p_c - p_n at a fluid-fluid face, p_c at an empty neighbour, -p_n in an empty cell).
    E_g is the sum of the E of the p_net values it takes; the divide, the difference, the subtraction and the final
    multiply are four roundings within u of s (|U1 / s| + |g| + E_g), so E_U = s_hi (E_g + gamma_4 (|U1| / s_lo + |g|
    + E_g)) + |g| (s_hi - s_lo); p = p_net s: s_hi E_p + u s_hi (|p_net| + E_p) + |p_net| (s_hi - s_lo).  Where
    VelocityUpdate sets 0 and where the wall mask zeroes a component, the GPU writes an exact 0 and E = 0, so the
    pattern of exact zeros is pinned with no extra rule.
Roundings of the float64 evaluation itself (2^-53 relative) are far below every u term and left out.

Cost: the float64 convolutions go through torch's conv3d in z chunks; a 128^3 'default' forward with its bound takes
about 10 s of CPU."""
import numpy as np
import torch
import torch.nn.functional as F

import oracle
from oracle import model as om
from oracle.model import DEFAULT_CHANNELS, model_inputs, network

U32 = 2.0 ** -24
U64 = 2.0 ** -53
SIGMOID_ULPS = 2.0 ** -20
KAPPA = {"tf32x3": 2.0 ** -16, "tf32": 2.0 ** -8}
TAIL_ULPS = 2.0 ** -20


def gamma(n):
    return n * U32 / (1.0 - n * U32)


def conv_f64(x, w, b=None, d=1):
    """oracle.model.conv64 (zero padding d (k - 1) / 2, dilation d) through torch's conv3d in z chunks, float64."""
    kz, k = w.shape[2], w.shape[4]
    pz, p = d * (kz - 1) // 2, d * (k - 1) // 2
    xt = F.pad(torch.from_numpy(np.ascontiguousarray(x, np.float64)), (0, 0, 0, 0, pz, pz))
    wt = torch.from_numpy(np.ascontiguousarray(w, np.float64))
    bt = None if b is None else torch.from_numpy(np.ascontiguousarray(b, np.float64))
    nz, ny, nx = x.shape[2:]
    step = max(1, (1 << 24) // (ny * nx * w.shape[1] * kz * k * k))
    out = [F.conv3d(xt[:, :, z0:min(nz, z0 + step) + 2 * pz], wt, bt, padding=(0, p, p), dilation=d)
           for z0 in range(0, nz, step)]
    return torch.cat(out, dim=2).numpy()


def tc_covered(model):
    """The graphs the tensor cores run (tfl_cnn_create_model_norm's tc_ok): the 3-D 'default' graph without sigmoid,
    single-bank or with banks split at stage 1 and joined at stage 3, no BN on a banked graph."""
    bk = model.get("banks")
    nl = len(model["layers"])
    return (model["is3D"] and nl == 5 and model.get("nonlinType", "relu") != "sigmoid" and
            not any(model.get(k) and any(v != 1 for v in model[k]) for k in ("pool", "up")) and
            (bk is None or bk["num"] == 1 or (bk["split_stage"] == 1 and bk["join_stage"] == 3 and
                                              not model.get("batchNorm"))))


class Bound:
    """oracle.model.F64's operations on (value, E) pairs for one arithmetic path: mode 'fp32', 'tf32x3' or 'tf32'."""

    def __init__(self, model, mode):
        assert mode == "fp32" or tc_covered(model), "the tensor cores do not run this graph"
        self.mode = mode
        bn = model.get("batchNorm")
        self.fold = mode != "fp32" and bn is not None and not bn["train"]
        self._fold_mag = None

    lift = staticmethod(lambda x: x)

    def kappa(self, li, w):
        if self.mode == "fp32":
            return gamma(w[0].size + 1)
        return KAPPA[self.mode] if w.shape[-1] == 3 else max(TAIL_ULPS, gamma(w[0].size + 1))

    def conv(self, x, w, b, is3d, d, li, relu):
        v, E = x
        wa = np.abs(w)
        kappa = self.kappa(li, w)
        m = np.abs(v) + E
        if self._fold_mag is not None:                       # a BN folded into these weights
            m, kappa = self._fold_mag, kappa + 2 * U32
            self._fold_mag = None
        y = conv_f64(v, w, b, d), kappa * conv_f64(m, wa, np.abs(b), d) + conv_f64(E, wa, None, d)
        return self.nonlin(y, "relu") if relu else y

    @staticmethod
    def shuffle(x, s, is3d):
        return tuple(om.shuffle(a, s, is3d) for a in x)

    @staticmethod
    def nonlin(x, kind):
        v, E = x
        y = om.nonlin(v, kind)
        if kind == "sigmoid":
            return y, E / 4 + SIGMOID_ULPS * y
        lo = np.clip(v + E, 0.0, E)                          # v + E <= 0: both clamp to exactly 0
        return y, (np.minimum(lo, np.clip(6.0 - v + E, 0.0, E)) if kind == "relu6" else lo)

    @staticmethod
    def pool(x, q, is3d, kind):
        v, E = x
        if kind == "max":
            return om.pool(v, q, is3d, "max"), om.pool(E, q, is3d, "max")
        m = om.pool(np.abs(v) + E, q, is3d, "avg")
        return om.pool(v, q, is3d, "avg"), om.pool(E, q, is3d, "avg") + gamma(q ** (3 if is3d else 2)) * m

    @staticmethod
    def up(x, r, is3d):
        return tuple(om.upsample(a, r, is3d) for a in x)

    @staticmethod
    def concat(hs):
        return np.concatenate([v for v, _ in hs], axis=1), np.concatenate([E for _, E in hs], axis=1)

    @staticmethod
    def add(hs):
        v = sum(h[0] for h in hs[1:]) + hs[0][0]
        E = sum(h[1] for h in hs[1:]) + hs[0][1]
        return v, E + gamma(len(hs) - 1) * sum(np.abs(h[0]) + h[1] for h in hs)

    def bn(self, x, e, train, li):
        v, E = x
        c_ = v.shape[1]
        s = lambda t: np.asarray(t, np.float64)[None, :, None, None, None]
        w = np.ones(c_) if e.get("weight") is None else np.asarray(e["weight"], np.float64)
        b = np.zeros(c_) if e.get("bias") is None else np.asarray(e["bias"], np.float64)
        eps = float(np.float32(e["eps"]))
        y = om.batch_norm(v, e, train)
        if not train:
            a = w / np.sqrt(np.asarray(e["running_var"], np.float64) + eps)
            c = b - np.asarray(e["running_mean"], np.float64) * a
            if self.fold and li in (2, 3):                   # BN3 into w4 / b4, BN4 into w5 / b5
                self._fold_mag = s(np.abs(a)) * (np.abs(v) + E) + s(np.abs(c))
                return y, s(np.abs(a)) * E
            return y, s(np.abs(a)) * E + gamma(3) * (s(np.abs(a)) * (np.abs(v) + E) + s(np.abs(c)))
        ax = (0, 2, 3, 4)
        N = v.size // c_
        mag = np.abs(v) + E
        mean = v.mean(axis=ax)
        sigma = np.sqrt(((v - s(mean)) ** 2).mean(axis=ax))
        fp64 = (N + 4) * U64
        dmean = E.mean(axis=ax) + fp64 * (mag.mean(axis=ax) + mag.max(axis=ax))
        dsigma = np.sqrt((E ** 2).mean(axis=ax))
        dvar64 = fp64 * 2 * ((mag ** 2).mean(axis=ax) + mag.max(axis=ax) ** 2)
        dsd = dsigma + np.sqrt(dvar64)
        sd = np.sqrt(sigma ** 2 + eps)
        sd_lo = np.sqrt(np.maximum(sigma - dsd, 0.0) ** 2 + eps)
        with np.errstate(divide="ignore", invalid="ignore"):
            a = np.where(sd > 0, w / sd, 0.0)
            da = np.where(sd_lo > 0, np.abs(w) * dsd / (sd * sd_lo), np.inf)
        aa = np.abs(a) + da
        cc = np.abs(b) + (np.abs(mean) + dmean) * aa
        Ey = s(aa) * (E + s(dmean)) + s(da) * np.abs(v - s(mean)) + gamma(3) * (s(aa) * mag + s(cc))
        return y, Ey


# ---------------------------------------------------------------------------------------------------------------
# Input block, scale, finish
# ---------------------------------------------------------------------------------------------------------------
def occupancy(be, flags):
    """tfluids.FlagsToOccupancy: 0 fluid, 1 obstacle.  The reference refuses any other flag value; the library writes
    -1 for them (cnn_input_channels, tfl_model_stages.cu), which Empty, Outflow and Stick cells get here."""
    f = flags.astype(np.int32)
    if np.isin(f, (1, 2)).all():
        return be.flagsToOccupancy(flags)
    return np.where(f == 1, 0.0, np.where(f == 2, 1.0, -1.0)).astype(np.float32)


def input_fields(be, pDiv, UDiv, flags):
    """The oracle's U1 (SetWallBcs as a mask multiply), div(U1) and the occupancy: bit-exact with the GPU."""
    U1 = np.ascontiguousarray(UDiv, np.float32).copy()
    be.setWallBcsForward(U1, flags, as_mask_multiply=True)
    return {"pDiv": np.asarray(pDiv, np.float32), "U1": U1, "div": be.velocityDivergenceForward(U1, flags),
            "occ": occupancy(be, flags)}


def _neighbours(f):
    f = np.float32(f)
    return np.array([np.nextafter(f, np.float32(-np.inf)), f, np.nextafter(f, np.float32(np.inf))], np.float32)


def scale_interval(field, func="std", threshold=1e-5):
    """[lo, hi] for one entry's scale: scale_from_sums (tfl_device.cuh) or the 'norm' formula of k_cnn_scale in
    float32 on the exact sums of field and of its float32 squares, each converted to float one float either side,
    the product-sum with and without contraction."""
    f = np.asarray(field, np.float32).ravel()
    s1 = f.astype(np.float64).sum()
    s2 = (f * f).astype(np.float64).sum()
    n = f.size
    th = np.float32(threshold)
    out = []
    for q in _neighbours(s2):
        if func == "norm":
            out.append(max(np.sqrt(q), th))
            continue
        for s in _neighbours(s1):
            ss = s * s
            for t in (q * np.float32(n) + np.float32(-1.0) * ss,
                      np.float32(float(q) * float(np.float32(n)) - float(ss))):
                t = t / np.float32(float(n) * float(n - 1))
                out.append(max(np.sqrt(np.float32(t)), th))
    return float(min(out)), float(max(out))


def network_input(fields, is3d, s_lo, s_hi, s_mid, inputChannels=None):
    """x0 (float64) and its bound for per-entry scales [b]: pDiv / s, U1 / s, div / s, occupancy."""
    ch = dict(DEFAULT_CHANNELS, **(inputChannels or {}))
    sm = np.asarray(s_mid, np.float64).reshape(-1, 1, 1, 1, 1)
    rho = ((np.asarray(s_hi, np.float64) - np.asarray(s_lo, np.float64)) / np.asarray(s_lo, np.float64))
    rho = rho.reshape(-1, 1, 1, 1, 1)
    xs, Es = [], []
    for key, on in (("pDiv", ch["pDiv"]), ("U1", ch["UDiv"]), ("div", ch["div"])):
        if on:
            x = fields[key].astype(np.float64) / sm
            xs.append(x)
            Es.append((U32 + rho) * np.abs(x))
    xs.append(fields["occ"].astype(np.float64))
    Es.append(np.zeros_like(xs[-1]))
    return np.concatenate(xs, axis=1), np.concatenate(Es, axis=1)


def _shift(a, axis):
    """a at i - 1 along `axis` (0 at i = 0, which is a border cell)."""
    out = np.zeros_like(a)
    dst, src = [slice(None)] * a.ndim, [slice(None)] * a.ndim
    dst[axis], src[axis] = slice(1, None), slice(None, -1)
    out[tuple(dst)] = a[tuple(src)]
    return out


def finish(be, U1, flags, pn, Epn, is3d, s_lo, s_hi, s_mid):
    """(p, Ep, U, EU): p = p_net s and U = setWallBcs((U1 / s - g) s) in float64 with their bounds (module
    docstring).  pn, Epn [b][1][z][y][x]; scales [b]."""
    B = U1.shape[0]
    r = lambda t: np.asarray(t, np.float64).reshape(B, 1, 1, 1)
    slo, shi, smid = r(s_lo), r(s_hi), r(s_mid)
    f = flags[:, 0].astype(np.int32)
    pc, Ec = pn[:, 0], Epn[:, 0]
    inner = np.zeros(f.shape, bool)
    if is3d:
        inner[:, 1:-1, 1:-1, 1:-1] = True
    else:
        inner[:, :, 1:-1, 1:-1] = True
    fluid = inner & ((f & 1) != 0)
    empty = inner & ~((f & 1) != 0) & ((f & 4) != 0) & ((f & 16) == 0)
    mask = np.ones(U1.shape, np.float32)
    be.setWallBcsForward(mask, flags, as_mask_multiply=True)
    U, EU = np.zeros(U1.shape), np.zeros(U1.shape)
    for a in range(U1.shape[1]):
        axis = 3 - a                                         # x, y, z in [b][z][y][x]
        fn, pnb, Enb = _shift(f, axis), _shift(pc, axis), _shift(Ec, axis)
        nbf, nbe = (fn & 1) != 0, (fn & 4) != 0
        g = np.where(fluid, np.where(nbf, pc - pnb, 0.0) + np.where(nbe, pc, 0.0), np.where(empty & nbf, -pnb, 0.0))
        Eg = np.where(fluid, np.where(nbf, Ec + Enb, 0.0) + np.where(nbe, Ec, 0.0), np.where(empty & nbf, Enb, 0.0))
        zero = (empty & ~nbf) | (mask[:, a] == 0)
        t = U1[:, a].astype(np.float64)
        U[:, a] = np.where(zero, 0.0, t - smid * g)
        EU[:, a] = np.where(zero, 0.0, shi * (Eg + gamma(4) * (np.abs(t) / slo + np.abs(g) + Eg))
                            + np.abs(g) * (shi - slo))
    p = pn * smid[:, None]
    Ep = shi[:, None] * (Epn + U32 * (np.abs(pn) + Epn)) + np.abs(pn) * (shi - slo)[:, None]
    return p, Ep, U, EU


# ---------------------------------------------------------------------------------------------------------------
# The whole forward
# ---------------------------------------------------------------------------------------------------------------
def scale_intervals(fields, model, threshold=1e-5):
    """Per entry (lo, hi) of the input scale (1 without normalizeInput)."""
    kw = model_inputs(model)
    B = fields["U1"].shape[0]
    if not kw["normalizeInput"]:
        return np.ones(B), np.ones(B)
    field = fields[{"UDiv": "U1", "pDiv": "pDiv", "div": "div"}[kw["normalizeInputChan"]]]
    iv = np.array([scale_interval(field[b], kw["normalizeInputFunc"], threshold) for b in range(B)])
    return iv[:, 0], iv[:, 1]


def p_net_bound(model, x0, E0, mode, pS=None, rho=0.0):
    """p_net [b][1][z][y][x] and its bound; pS (pDiv / s_mid, float64) with addPressureSkip, rho [b] the scale
    interval's relative width (pDiv / s_gpu is within rho |pS| of pS)."""
    ops = Bound(model, mode)
    if pS is None:
        return network(model, (x0, E0), ops)
    hv, hE = network(model, (x0, E0), ops, hidden=True)
    w, b = model["layers"][-1]
    body_v, body_E = ops.conv((hv, hE), w[:, :-1], b, model["is3D"], 1, len(model["layers"]) - 1, False)
    skip = float(w[0, -1].ravel()[0]) * pS
    rho = np.asarray(rho, np.float64).reshape(-1, 1, 1, 1, 1)
    return body_v + skip, body_E + gamma(3) * (np.abs(body_v) + body_E + np.abs(skip)) + rho * np.abs(skip)


def forward_bound(be, model, pDiv, UDiv, flags, mode, scale=None, threshold=1e-5):
    """The float64 forward of lib/model.lua:27-401 and its per-voxel bound on the GPU's result in `mode`.  scale: the
    GPU's per-entry scales (ProjectionModel.forward(return_scale=True)), or None for the scale interval.
    Returns dict(p, Ep, U, EU, s_lo, s_hi): p [b][1][z][y][x], U [b][nc][z][y][x], float64."""
    kw = model_inputs(model)
    fields = input_fields(be, pDiv, UDiv, flags)
    lo, hi = scale_intervals(fields, model, threshold)
    if scale is None:
        s_lo, s_hi, s_mid = lo, hi, (lo + hi) / 2
    else:
        s_lo = s_hi = s_mid = np.asarray(scale, np.float64)
    x0, E0 = network_input(fields, model["is3D"], s_lo, s_hi, s_mid, kw["inputChannels"])
    pS = None
    if kw["addPressureSkip"]:
        pS = fields["pDiv"].astype(np.float64) / np.asarray(s_mid, np.float64).reshape(-1, 1, 1, 1, 1)
    pn, Epn = p_net_bound(model, x0, E0, mode, pS, (np.asarray(s_hi) - np.asarray(s_lo)) / np.asarray(s_lo))
    p, Ep, U, EU = finish(be, fields["U1"], flags, pn, Epn, model["is3D"], s_lo, s_hi, s_mid)
    return {"p": p, "Ep": Ep, "U": U, "EU": EU, "s_lo": lo, "s_hi": hi}


def excess(got, want, E):
    """(max err / E, worst index, err, E there); err / E is inf where E = 0 and got != want."""
    err = np.abs(np.asarray(got, np.float64) - want)
    with np.errstate(divide="ignore", invalid="ignore"):
        ratio = np.where(err == 0, 0.0, err / E)
    worst = np.unravel_index(np.argmax(ratio), ratio.shape)
    return float(ratio[worst]), worst, float(err[worst]), float(E[worst])


def check(what, got, want, E):
    """|got - want| <= E at every voxel; returns max err / E."""
    r, worst, err, bound = excess(got, want, E)
    assert r <= 1.0, "%s: %d voxels over the bound; worst %s: err %.3e bound %.3e (err/E %.3g)" % (
        what, int((np.abs(np.asarray(got, np.float64) - want) > E).sum()), worst, err, bound, r)
    return r


def projection_reference(state, mconf, gm, mnp):
    """The float64 projection of one step from `state` (GPU tensors, left as they are) on the scale interval: the
    operator sequence up to the projection and setConstVals, forward_bound, then the U BCs (x inv + bc: E |inv| plus
    two roundings) and the +-1e6 clamp (1-Lipschitz)."""
    from fluidnet_b200 import simulate
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
