"""Batch normalization (addBatchNorm) and nonlinType 'relu6' of torch/lib/model.lua:316-350 and
lib/model_utils.lua:20-62 on the CPU, for the tests: a float64 restatement of the whole network for every graph the
library builds -- 'default' / 'tog' / 'yang', 'mres' and 'dilate' banks, any input block, with or without the pressure
skip.

Facts it restates:
  * Every stage but the last, and every bank of a banked stage, is convolution -> non-linearity -> pooling (psize > 1)
    -> BN over its osize channels.  The non-linearity and BN come after the pixel shuffle of an upsampling stage, at
    the stage's output resolution; an 'mres' bank's BN runs at that bank's resolution with its own parameters, before
    the join; a 'dilate' bank's at full resolution.  The final convolution has no BN.
  * A module saved with train = true (the nn.Module default: the reference's simulators never call evaluate())
    normalises with batch statistics: per channel, the mean and the biased variance over all batch entries and
    voxels, y = (x - mean) / sqrt(var + eps) w + b, with 1 / sqrt(var + eps) taken as 0 where var + eps == 0 (THNN).
    train = false: y = (x - running_mean) / sqrt(running_var + eps) w + b.  Without batchNormAffine w = 1, b = 0.
  * 'relu6' is nn.ReLU6, min(max(x, 0), 6).

`model_forward_bn` has oracle.model_forward's signature plus the input-block keywords of
tests/inputs_oracle.model_forward_inputs; the model is a synth.make_model dict whose "batchNorm" (may be missing) is
in the form of model.ProjectionModel's keyword.  The input block and the velocity update go through the oracle backend
as in tests/inputs_oracle.py; the network runs in float64 and is rounded to float32 once, at its output.
tests/test_oracle_model_bn.py pins it on torch.nn.functional."""
import numpy as np

from inputs_oracle import model_input


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


def _pool(x, q, is3d, kind):
    b_, c_, z_, y_, x_ = x.shape
    qz = q if is3d else 1
    v = x.reshape(b_, c_, z_ // qz, qz, y_ // q, q, x_ // q, q)
    return v.max(axis=(3, 5, 7)) if kind == "max" else v.mean(axis=(3, 5, 7))


def _shuffle(x, s_, is3d):
    b_, ct, z_, y_, x_ = x.shape
    if is3d:
        no = ct // s_ ** 3
        x = x.reshape(b_, no, s_, s_, s_, z_, y_, x_).transpose(0, 1, 5, 2, 6, 3, 7, 4)
        return np.ascontiguousarray(x).reshape(b_, no, z_ * s_, y_ * s_, x_ * s_)
    no = ct // s_ ** 2
    x = x.reshape(b_, no, s_, s_, z_, y_, x_).transpose(0, 1, 4, 5, 2, 6, 3)
    return np.ascontiguousarray(x).reshape(b_, no, z_, y_ * s_, x_ * s_)


def _rep(a, r, is3d):
    """Nearest up-sampling by r (the join of an 'mres' bank)."""
    return np.repeat(np.repeat(np.repeat(a, r, 2), r, 3), r, 4) if is3d else np.repeat(np.repeat(a, r, 3), r, 4)


class F64:
    """The float64 operations `stage` and `network` compose.  tests/network_bound.py substitutes operations on
    (value, error bound) pairs and a float32 emulation of the library with the same signatures; `li` is the stage
    index (0-based) of the convolution or BN it belongs to."""
    lift = staticmethod(lambda x: np.asarray(x, np.float64))
    conv = staticmethod(lambda x, w, b, is3d, d, li: conv64(x, w, b, is3d, d))
    shuffle = staticmethod(_shuffle)
    nonlin = staticmethod(nonlin)
    pool = staticmethod(_pool)
    bn = staticmethod(lambda x, e, train, li: batch_norm(x, e, train))
    up = staticmethod(_rep)
    concat = staticmethod(lambda hs: np.concatenate(hs, axis=1))
    add = staticmethod(lambda hs: sum(hs[1:], hs[0]))


def stage(model, li, w, b, x, d=1, bn=None, ops=F64):
    """One stage of model.lua:320-350: convolution (dilated by d) -> shuffle -> non-linearity -> pooling -> BN."""
    is3d = model["is3D"]
    nl = len(model["layers"])
    pool = model.get("pool") or [1] * nl
    up = model.get("up") or [1] * nl
    x = ops.conv(x, w, b, is3d, d, li)
    if up[li] > 1:
        x = ops.shuffle(x, up[li], is3d)
    if li < nl - 1:
        x = ops.nonlin(x, model.get("nonlinType", "relu"))
    if pool[li] > 1:
        x = ops.pool(x, pool[li], is3d, model.get("poolType", "avg"))
    if bn is not None:
        x = ops.bn(x, bn, model["batchNorm"]["train"], li)
    return x


def network(model, x, hidden=False, ops=F64):
    """The stages on the network input x -> p_net [b][1][z][y][x] (float64); hidden=True stops before the last
    convolution and returns its input.  `ops` (default F64) supplies the operations."""
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
        hl = [stage(model, li, w, b, h, 2 ** i if dil else 1, e, ops)
              for i, ((w, b), h, e) in enumerate(zip(convs, hl, bns))]
    assert len(hl) == 1
    return hl[0]


def model_forward_bn(be, model, pDiv, UDiv, flags, threshold=1e-5, inputChannels=None, normalizeInput=True,
                     normalizeInputFunc="std", normalizeInputChan="UDiv", addPressureSkip=False):
    """lib/model.lua:27-401 with batch normalization and relu6.  Returns (p, U, scale)."""
    x, pS, US, sc, scales = model_input(be, pDiv, UDiv, flags, threshold, inputChannels, normalizeInput,
                                        normalizeInputFunc, normalizeInputChan)
    if addPressureSkip:                                                 # :357-361 JoinTable(2)({hl, pDiv})
        w, b = model["layers"][-1]
        h = np.concatenate([network(model, x, hidden=True), np.asarray(pS, np.float64)], axis=1)
        p = conv64(h, w, b, model["is3D"]).astype(np.float32)
    else:
        p = network(model, x).astype(np.float32)
    U2 = np.ascontiguousarray(US.copy())
    be.velocityUpdateForward(U2, flags, p)
    if normalizeInput:
        p = (p * sc).astype(np.float32)
        U2 = np.ascontiguousarray((U2 * sc).astype(np.float32))
    be.setWallBcsForward(U2, flags, as_mask_multiply=True)
    return p, U2, scales


def model_forward_of_model(be, model, pDiv, UDiv, flags, threshold=1e-5):
    """oracle.model_forward's signature with the input block read from model["inputs"], so that oracle.simulate can
    run a BN model."""
    return model_forward_bn(be, model, pDiv, UDiv, flags, threshold, **(model.get("inputs") or {}))
