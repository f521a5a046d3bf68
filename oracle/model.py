"""TEST INFRASTRUCTURE ONLY (see oracle/__init__.py) -- the projection network of torch/lib/model.lua:27-401.

`model_forward` is the whole forward: input block, network, velocity update.  `network` is its one stage loop; an
operations table supplies the arithmetic: `Float32Ops(be)` is the oracle's float32 evaluation (what oracle.simulate
runs), `F64` evaluates the network in float64 and rounds to float32 once, at its output, and tests/network_bound.py
runs the same loop on (value, error bound) pairs.  The model is a fluidnet_b200.synth.make_model dict: "is3D",
"layers" [(weight, bias), ...; a banked stage holds one pair per bank], and optionally "pool", "up", "poolType",
"nonlinType", "banks", "inputs" (the keywords of model.ProjectionModel) and "batchNorm".

Facts it restates:
  * Input block (model.lua:27-150).  U1 = SetWallBcs(UDiv) as a mask multiply (:81-84) and div = div(U1) (:86-89).
    With normalizeInput each entry's scale is nn.StandardDeviation ('std', :96-97) or Power(2), Sum, Sqrt ('norm',
    :98-102, float64 sums) of the field normalizeInputChan (:108-116), clamped below at the threshold (:106), and
    pDiv, U1 and div are divided by it (:119-130); without it there is no scale node (:92): the scale is 1, and
    dividing and multiplying by 1 are exact.  The network input is nn.JoinTable(2) of the inputChannels in the order
    pDiv, UDiv, div, occupancy (:133-150; default set lib/default_conf.lua:76-81).
  * Stages (model.lua:320-350).  Every stage is convolution -> pixel shuffle (an upsampling stage,
    *_convolution_upsample.lua) -> non-linearity -> pooling (psize > 1, cudnn avg / max) -> BN over its osize
    channels; the last stage is the convolution alone.  'relu6' is nn.ReLU6, min(max(x, 0), 6).
  * 'mres' banks (model.lua:252-361).  At banksSplitStage the hidden layer is split into a pyramid: bank i is a 2x
    average pool of bank i-1.  The stages in between run one convolution stage per bank.  At banksJoinStage bank i is
    upsampled nearest by 2^(i-1), and the banks are concatenated along the channels in bank order (nn.JoinTable) or
    summed left to right (nn.CAddTable).
  * 'dilate' banks.  At the split every bank takes the hidden layer as it is (model.lua:279-285); bank i's
    convolutions are dilated by 2^(i-1) on every axis with zero padding 2^(i-1) (k-1)/2, so the grid is kept
    (nn.{Spatial,Volumetric}DilatedConvolution, lib/model_utils.lua:122-146); the join concatenates or sums them
    without upsampling (model.lua:300-318).
  * Batch normalization (addBatchNorm, model.lua:316-350, lib/model_utils.lua:20-62).  An 'mres' bank's BN runs at
    that bank's resolution with its own parameters, before the join; a 'dilate' bank's at full resolution.  A module
    saved with train = true (the nn.Module default: the reference's simulators never call evaluate()) normalises with
    batch statistics: per channel, the mean and the biased variance over all batch entries and voxels,
    y = (x - mean) / sqrt(var + eps) w + b, with 1 / sqrt(var + eps) taken as 0 where var + eps == 0 (THNN).
    train = false: y = (x - running_mean) / sqrt(running_var + eps) w + b.  Without batchNormAffine w = 1, b = 0.
  * addPressureSkip (model.lua:357-361): JoinTable(2)({hl, pDiv}), the scaled pDiv joined to the hidden layer before
    the last convolution.
  * Output (:380-390): VelocityUpdate on the scaled U1, then p and U multiplied by the scale, then the wall mask.
tests/test_oracle_model_{graph,banks,dilate,inputs,bn}.py pin this on numpy / torch.nn.functional in float64."""
import numpy as np

DEFAULT_INPUTS = dict(inputChannels=None, normalizeInput=True, normalizeInputFunc="std", normalizeInputChan="UDiv",
                      addPressureSkip=False)
DEFAULT_CHANNELS = {"pDiv": True, "UDiv": False, "div": True, "flags": True}      # lib/default_conf.lua:76-81


def model_inputs(model):
    """The input-block keywords of a model dict, with their defaults."""
    return dict(DEFAULT_INPUTS, **(model.get("inputs") or {}))


def model_input(be, model, pDiv, UDiv, flags, threshold=1e-5):
    """The network input x, the scaled pDiv and UDiv, and the scale through the backend `be`.
    Returns (x, pS, US, sc [b,1,1,1,1], scales [b])."""
    kw = model_inputs(model)
    ch = dict(DEFAULT_CHANNELS, **(kw["inputChannels"] or {}))
    U1 = UDiv.copy()
    be.setWallBcsForward(U1, flags, as_mask_multiply=True)              # model.lua:81-84
    div = be.velocityDivergenceForward(U1, flags)                       # :86-89
    b = U1.shape[0]
    scales = np.ones(b, np.float32)
    if kw["normalizeInput"]:                                            # :92-117
        field = {"UDiv": U1, "pDiv": pDiv, "div": div}[kw["normalizeInputChan"]]
        for ib in range(b):
            if kw["normalizeInputFunc"] == "std":
                s = np.float32(be.sampleStd(field[ib]))
            else:
                f = np.asarray(field[ib], np.float32)
                s = np.float32(np.sqrt(np.sum((f * f).astype(np.float64))))
            scales[ib] = max(s, np.float32(threshold))
    sc = scales.reshape(b, 1, 1, 1, 1)
    pS = (pDiv / sc).astype(np.float32)                                 # :119-130
    US = (U1 / sc).astype(np.float32)
    divS = (div / sc).astype(np.float32)
    occ = be.flagsToOccupancy(flags)                                    # :144-147
    chans = [c for c, on in ((pS, ch["pDiv"]), (US, ch["UDiv"]), (divS, ch["div"]), (occ, ch["flags"])) if on]
    x = np.ascontiguousarray(np.concatenate(chans, axis=1))             # :133-150
    return x, pS, US, sc, scales


def conv64(x, w, b, is3d, d=1):
    """Zero-padded stride-1 cross-correlation dilated by d (padding d (k-1)/2), float64 throughout."""
    cout, cin, kz, k, _ = w.shape
    pz, p = d * (kz - 1) // 2, d * (k - 1) // 2
    B, _, Z, Y, X = x.shape
    xp = np.zeros((B, cin, Z + 2 * pz, Y + 2 * p, X + 2 * p))
    xp[:, :, pz:pz + Z, p:p + Y, p:p + X] = x
    acc = np.zeros((B, cout, Z, Y, X)) + b.astype(np.float64)[None, :, None, None, None]
    w64 = w.astype(np.float64)
    for tz in range(kz):
        for ty in range(k):
            for tx in range(k):
                sl = xp[:, :, tz * d:tz * d + Z, ty * d:ty * d + Y, tx * d:tx * d + X]
                acc += np.einsum("oc,bczyx->bozyx", w64[:, :, tz, ty, tx], sl)
    return acc


def nonlin(x, kind):
    if kind == "sigmoid":
        return 1.0 / (1.0 + np.exp(-x))
    if kind == "relu6":
        return np.minimum(np.maximum(x, 0.0), 6.0)
    return np.maximum(x, 0.0)


def batch_norm(x, e, train):
    """One {Spatial,Volumetric}BatchNormalization module on x [B][c][Z][Y][X] (float64)."""
    c = x.shape[1]
    w = np.ones(c) if e.get("weight") is None else np.asarray(e["weight"], np.float64)
    b = np.zeros(c) if e.get("bias") is None else np.asarray(e["bias"], np.float64)
    eps = float(np.float32(e["eps"]))
    if train:
        mean = x.mean(axis=(0, 2, 3, 4))
        var = ((x - mean[None, :, None, None, None]) ** 2).mean(axis=(0, 2, 3, 4))
        ve = var + eps
        invstd = np.where(ve == 0.0, 0.0, 1.0 / np.sqrt(np.where(ve == 0.0, 1.0, ve)))
    else:
        mean = np.asarray(e["running_mean"], np.float64)
        invstd = 1.0 / np.sqrt(np.asarray(e["running_var"], np.float64) + eps)
    s = lambda v: v[None, :, None, None, None]
    return (x - s(mean)) * s(invstd * w) + s(b)


def pool(x, q, is3d, kind):
    b_, c_, z_, y_, x_ = x.shape
    qz = q if is3d else 1
    v = x.reshape(b_, c_, z_ // qz, qz, y_ // q, q, x_ // q, q)
    return v.max(axis=(3, 5, 7)) if kind == "max" else v.mean(axis=(3, 5, 7))


def shuffle(x, s_, is3d):
    b_, ct, z_, y_, x_ = x.shape
    if is3d:
        no = ct // s_ ** 3
        x = x.reshape(b_, no, s_, s_, s_, z_, y_, x_).transpose(0, 1, 5, 2, 6, 3, 7, 4)
        return np.ascontiguousarray(x).reshape(b_, no, z_ * s_, y_ * s_, x_ * s_)
    no = ct // s_ ** 2
    x = x.reshape(b_, no, s_, s_, z_, y_, x_).transpose(0, 1, 4, 5, 2, 6, 3)
    return np.ascontiguousarray(x).reshape(b_, no, z_, y_ * s_, x_ * s_)


def upsample(a, r, is3d):
    """Nearest up-sampling by r (the join of an 'mres' bank)."""
    return np.repeat(np.repeat(np.repeat(a, r, 2), r, 3), r, 4) if is3d else np.repeat(np.repeat(a, r, 3), r, 4)


class F64:
    """The float64 operations `network` composes.  `li` is the stage index (0-based) of the convolution or BN it
    belongs to; `relu` asks the convolution for the stage's ReLU (Float32Ops fuses it into the backend's)."""
    lift = staticmethod(lambda x: np.asarray(x, np.float64))

    @staticmethod
    def conv(x, w, b, is3d, d, li, relu):
        y = conv64(x, w, b, is3d, d)
        return nonlin(y, "relu") if relu else y

    shuffle = staticmethod(shuffle)
    nonlin = staticmethod(nonlin)
    pool = staticmethod(pool)
    bn = staticmethod(lambda x, e, train, li: batch_norm(x, e, train))
    up = staticmethod(upsample)
    concat = staticmethod(lambda hs: np.concatenate(hs, axis=1))
    add = staticmethod(lambda hs: sum(hs[1:], hs[0]))


class Float32Ops(F64):
    """The oracle's float32 network through the backend `be`: undilated convolutions are be.conv (double sums rounded
    to float) with the stage's ReLU fused there, so a -0 keeps its sign as orc_conv keeps it; a dilated convolution,
    the non-linearities and the pools are evaluated in float64 on the float32 values and rounded once (an average
    pool is a float64 sum divided by the count); the join moves float32 values or sums them left to right in
    float32.  There is no float32 batch normalization."""

    def __init__(self, be):
        self.be = be

    lift = staticmethod(lambda x: np.asarray(x, np.float32))

    def conv(self, x, w, b, is3d, d, li, relu):
        if d == 1:
            return self.be.conv(x, w, b, is3d, relu)
        return F64.conv(x, w, b, is3d, d, li, relu).astype(np.float32)

    nonlin = staticmethod(lambda x, kind: nonlin(x.astype(np.float64), kind).astype(np.float32))
    pool = staticmethod(lambda x, q, is3d, kind: pool(x.astype(np.float64), q, is3d, kind).astype(np.float32))

    def bn(self, x, e, train, li):
        raise NotImplementedError("the oracle has no float32 batch normalization: use model_forward(f64=True)")


def _stage(model, li, w, b, x, d, bn, ops):
    """One stage of model.lua:320-350: convolution (dilated by d) -> shuffle -> non-linearity -> pooling -> BN."""
    is3d = model["is3D"]
    nl = len(model["layers"])
    psize = model.get("pool") or [1] * nl
    usize = model.get("up") or [1] * nl
    kind = model.get("nonlinType", "relu") if li < nl - 1 else None
    relu = kind == "relu" and usize[li] == 1 and psize[li] == 1        # nothing between: the convolution takes it
    x = ops.conv(x, w, b, is3d, d, li, relu)
    if usize[li] > 1:
        x = ops.shuffle(x, usize[li], is3d)
    if kind is not None and not relu:
        x = ops.nonlin(x, kind)
    if psize[li] > 1:
        x = ops.pool(x, psize[li], is3d, model.get("poolType", "avg"))
    if bn is not None:
        x = ops.bn(x, bn, model["batchNorm"]["train"], li)
    return x


def network(model, x, ops, hidden=False):
    """The stages on the network input x -> p_net [b][1][z][y][x] in the arithmetic of `ops`; hidden=True stops
    before the last convolution and returns its input."""
    is3d = model["is3D"]
    banks = model.get("banks")
    n = banks["num"] if banks else 1
    s, j = (banks["split_stage"], banks["join_stage"]) if banks else (0, 0)
    dil = bool(banks) and banks.get("type") == "dilate"
    bnl = (model.get("batchNorm") or {}).get("layers")
    nl = len(model["layers"])
    hl = [ops.lift(x)]
    for li, layer in enumerate(model["layers"]):
        lid = li + 1
        if n > 1 and lid == s:
            hl = [hl[0]] * n if dil else [hl[0]]
            for i in range(1, n if not dil else 1):
                hl.append(ops.pool(hl[i - 1], 2, is3d, "avg"))
        if n > 1 and lid == j:
            ups = hl if dil else [hl[0]] + [ops.up(hl[i], 2 ** i, is3d) for i in range(1, n)]
            hl = [ops.concat(ups)] if banks["aggregate"] == "concat" else [ops.add(ups)]
        if hidden and li == nl - 1:
            return hl[0]
        convs = layer if isinstance(layer[0], (tuple, list)) else [layer]
        bns = [None] * len(convs)
        if bnl is not None and li < nl - 1:
            bns = bnl[li] if isinstance(bnl[li], (tuple, list)) else [bnl[li]]
        assert len(convs) == len(hl) == len(bns)
        hl = [_stage(model, li, w, b, h, 2 ** i if dil else 1, e, ops)
              for i, ((w, b), h, e) in enumerate(zip(convs, hl, bns))]
    assert len(hl) == 1
    return hl[0]


def model_forward(be, model, pDiv, UDiv, flags, threshold=1e-5, f64=False):
    """lib/model.lua:27-401 through the backend `be` (an oracle.Oracle or oracle.Reference), the network in
    float32 (Float32Ops) or, with f64, in float64 (F64).  Returns (p, U, scale [b]), float32."""
    x, pS, US, sc, scales = model_input(be, model, pDiv, UDiv, flags, threshold)
    ops = F64 if f64 else Float32Ops(be)
    if model_inputs(model)["addPressureSkip"]:                          # :357-361
        w, b = model["layers"][-1]
        h = ops.concat([network(model, x, ops, hidden=True), ops.lift(pS)])
        p = ops.conv(h, w, b, model["is3D"], 1, len(model["layers"]) - 1, False)
    else:
        p = network(model, x, ops)
    p = np.ascontiguousarray(p, np.float32)
    U = np.ascontiguousarray(US.copy())
    be.velocityUpdateForward(U, flags, p)                               # :380
    p = (p * sc).astype(np.float32)                                     # :384-387
    U = np.ascontiguousarray((U * sc).astype(np.float32))
    be.setWallBcsForward(U, flags, as_mask_multiply=True)               # :390
    return p, U, scales
