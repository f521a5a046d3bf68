"""The CPU restatement of batch normalization and relu6 (tests/bn_oracle.py, lib/model.lua:316-350,
lib/model_utils.lua:20-62) against an independent float64 evaluation with torch.nn.functional: conv{2,3}d (dilated for
'dilate' banks), the pixel shuffle, hardtanh(0, 6) / relu / sigmoid, avg / max pooling, batch_norm(training=True)
for modules saved with train = true and batch_norm(training=False) with the running statistics otherwise, avg_pool
pyramids and nearest upsampling for 'mres' banks.  The GPU path is then compared with the restatement."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import oracle
from bn_oracle import batch_norm, model_forward_bn, network
from inputs_oracle import model_forward_inputs, model_input
from fluidnet_b200 import synth


def torch_stage(t, model, li, w, b, d, bn):
    is3d = model["is3D"]
    nl = len(model["layers"])
    pool = model.get("pool") or [1] * nl
    up = model.get("up") or [1] * nl
    wt, bt = torch.from_numpy(w).double(), torch.from_numpy(b).double()
    pad = d * (w.shape[-1] - 1) // 2
    t = F.conv3d(t, wt, bt, padding=pad, dilation=d) if is3d else F.conv2d(t, wt[:, :, 0], bt, padding=pad, dilation=d)
    s = up[li]
    if s > 1:
        if is3d:
            bsz, ct, dd, h, w_ = t.shape
            no = ct // s ** 3
            out = torch.empty(bsz, no, dd * s, h * s, w_ * s, dtype=t.dtype)
            for st in range(s):
                for sh in range(s):
                    for sw in range(s):
                        out[:, :, st::s, sh::s, sw::s] = t[:, torch.arange(no) * s ** 3 + (st * s + sh) * s + sw]
            t = out
        else:
            t = F.pixel_shuffle(t, s)
    if li < nl - 1:
        kind = model.get("nonlinType", "relu")
        t = torch.sigmoid(t) if kind == "sigmoid" else (F.hardtanh(t, 0.0, 6.0) if kind == "relu6" else F.relu(t))
    if pool[li] > 1:
        if model.get("poolType", "avg") == "max":
            t = (F.max_pool3d if is3d else F.max_pool2d)(t, pool[li])
        else:
            t = (F.avg_pool3d if is3d else F.avg_pool2d)(t, pool[li])
    if bn is not None:
        c = t.shape[1]
        tt = lambda v, dflt: torch.full((c,), dflt, dtype=torch.float64) if v is None else torch.from_numpy(
            np.asarray(v, np.float64))
        t = F.batch_norm(t, tt(bn["running_mean"], 0), tt(bn["running_var"], 1), tt(bn.get("weight"), 1.0),
                         tt(bn.get("bias"), 0.0), training=model["batchNorm"]["train"], eps=float(np.float32(bn["eps"])))
    return t


def torch_network(x, model):
    is3d = model["is3D"]
    bk = model.get("banks")
    n, s, j = (bk["num"], bk["split_stage"], bk["join_stage"]) if bk else (1, 0, 0)
    dil = bool(bk) and bk.get("type") == "dilate"
    bnl = model["batchNorm"]["layers"]
    nl = len(model["layers"])
    t = torch.from_numpy(x).double()
    if not is3d:
        t = t[:, :, 0]
    hl = [t]
    for li, layer in enumerate(model["layers"]):
        if n > 1 and li + 1 == s:
            if dil:
                hl = hl * n
            else:
                for i in range(1, n):
                    hl.append((F.avg_pool3d if is3d else F.avg_pool2d)(hl[-1], 2))
        if n > 1 and li + 1 == j:
            ups = hl if dil else [hl[0]] + [F.interpolate(h, scale_factor=2 ** i, mode="nearest")
                                            for i, h in enumerate(hl) if i > 0]
            hl = [torch.cat(ups, dim=1)] if bk["aggregate"] == "concat" else [sum(ups[1:], ups[0])]
        convs = layer if isinstance(layer, list) else [layer]
        bns = [None] * len(convs) if li == nl - 1 else (bnl[li] if isinstance(bnl[li], list) else [bnl[li]])
        hl = [torch_stage(h, model, li, w, b, 2 ** i if dil else 1, e)
              for i, ((w, b), h, e) in enumerate(zip(convs, hl, bns))]
    t = hl[0]
    if not is3d:
        t = t[:, :, None]
    return t.numpy()


def banks(num, agg, kind="mres", s=1, j=3):
    return {"num": num, "split_stage": s, "join_stage": j, "aggregate": agg, "type": kind}


# (is3d, model_type, banks, (nz, ny, nx))
GRAPHS = {
    "3d-default": (True, "default", None, (6, 7, 9)),
    "3d-tog": (True, "tog", None, (8, 8, 12)),
    "3d-yang": (True, "yang", None, (5, 6, 7)),
    "3d-mres-n2-concat": (True, "default", banks(2, "concat"), (8, 8, 12)),
    "3d-mres-n3-add": (True, "default", banks(3, "add"), (8, 12, 8)),
    "3d-dilate-n2-concat": (True, "default", banks(2, "concat", "dilate"), (5, 7, 9)),
    "3d-dilate-n3-add-s2j4": (True, "default", banks(3, "add", "dilate", 2, 4), (6, 5, 11)),
    "2d-default": (False, "default", None, (1, 11, 13)),
    "2d-tog": (False, "tog", None, (1, 16, 24)),
    "2d-yang": (False, "yang", None, (1, 12, 9)),
    "2d-mres-n2-add": (False, "default", banks(2, "add"), (1, 16, 12)),
    "2d-dilate-n3-concat": (False, "default", banks(3, "concat", "dilate"), (1, 9, 15)),
}


def bn_model(is3d, model_type, bk, train, affine=True, relu6=False, seed=4321):
    m = synth.make_model(is3d, seed=seed, model_type=model_type, banks=bk,
                         batch_norm={"train": train, "affine": affine})
    if relu6:
        m["nonlinType"] = "relu6"
        # values well past 6 after the first stage: the clamp is exercised
        w, b = m["layers"][0] if not isinstance(m["layers"][0], list) else m["layers"][0][0]
        w *= np.float32(30.0)
    return m


def network_input(nb, shape, is3d, seed):
    rs = np.random.RandomState(seed)
    c = 3
    x = rs.uniform(-1, 1, (nb, c) + shape).astype(np.float32)
    x[:, 2] = (x[:, 2] > -0.6).astype(np.float32)        # occupancy-like channel
    return x


@pytest.mark.parametrize("variant", ["train", "eval", "train-noaffine-relu6", "eval-relu6"])
@pytest.mark.parametrize("graph", list(GRAPHS))
def test_bn_network_matches_torch(graph, variant):
    is3d, model_type, bk, shape = GRAPHS[graph]
    train = variant.startswith("train")
    relu6 = "relu6" in variant and model_type != "yang"
    model = bn_model(is3d, model_type, bk, train, affine="noaffine" not in variant, relu6=relu6)
    x = network_input(2, shape, is3d, 17)
    got = network(model, x)
    want = torch_network(x, model)
    assert got.shape == (2, 1) + shape
    assert np.abs(got - want).max() <= 1e-10 * max(np.abs(want).max(), 1.0)


def test_relu6_clamps_in_the_restatement():
    """The first stage of a relu6 model really produces values above 6 before the clamp (so the GPU comparison
    exercises it)."""
    model = bn_model(True, "default", None, True, relu6=True)
    x = network_input(1, (6, 7, 9), True, 3)
    from bn_oracle import conv64
    w, b = model["layers"][0]
    pre = conv64(x.astype(np.float64), w, b, True)
    assert pre.max() > 6.0 and pre.min() < 0.0


def test_batch_norm_dead_channel_and_train_coupling():
    """var + eps == 0 gives invstd 0, so the channel becomes its bias; batch statistics couple the entries, running
    statistics do not."""
    x = np.zeros((2, 2, 3, 4, 5))
    x[:, 1] = np.random.RandomState(0).rand(2, 3, 4, 5)
    e = {"weight": np.array([2.0, 1.5]), "bias": np.array([0.25, -0.5]), "running_mean": np.zeros(2),
         "running_var": np.ones(2), "eps": 0.0}
    y = batch_norm(x, e, True)
    assert (y[:, 0] == 0.25).all()
    x2 = x.copy()
    x2[1, 1] += 1.0
    assert not np.array_equal(batch_norm(x2, e, True)[0, 1], y[0, 1])
    assert np.array_equal(batch_norm(x2, e, False)[0], batch_norm(x, e, False)[0])


@pytest.mark.parametrize("skip", [False, True])
def test_identity_bn_is_the_model_without_bn(skip):
    """Running statistics with w = 1, b = 0, mean 0, var 1 - eps is the identity: model_forward_bn then equals the
    input-block restatement (float32 convolutions) to float32 rounding, with and without the pressure skip."""
    orc = oracle.Oracle()
    inputs = {"addPressureSkip": True} if skip else None
    model = synth.make_model(True, inputs=inputs, batch_norm={"train": False})
    for e in model["batchNorm"]["layers"]:
        e.update(weight=np.ones(8, np.float32), bias=np.zeros(8, np.float32), running_mean=np.zeros(8, np.float32),
                 running_var=np.full(8, 1.0 - 1e-4, np.float32), eps=1e-4)
    flags = synth.make_flags(9, 8, 7, True, nb=2, geometry=False)
    U = synth.make_smooth_velocity(flags, True, amp=1.0)
    orc.setWallBcsForward(U, flags)
    p0 = (synth.make_density(flags, seed=5) - np.float32(0.5)) * np.float32(0.1)
    kw = model.get("inputs") or {}
    a = model_forward_bn(orc, model, p0, U, flags, **kw)
    b = model_forward_inputs(orc, dict(model, batchNorm=None), p0, U, flags, **kw)
    for u, v in zip(a, b):
        assert np.abs(u - v).max() <= 1e-5 * max(np.abs(v).max(), 1e-3)


def test_pressure_skip_with_bn_matches_torch():
    """The skip joins the scaled pDiv to the BN'd hidden layer before the last 1x1 convolution."""
    orc = oracle.Oracle()
    model = synth.make_model(True, inputs={"addPressureSkip": True}, batch_norm={"train": True})
    flags = synth.make_flags(8, 7, 6, True, nb=2, geometry=False)
    U = synth.make_smooth_velocity(flags, True, amp=1.0)
    orc.setWallBcsForward(U, flags)
    p0 = (synth.make_density(flags, seed=5) - np.float32(0.5)) * np.float32(0.1)
    p, _, scale = model_forward_bn(orc, model, p0, U, flags, addPressureSkip=True)
    x, pS, _, sc, _ = model_input(orc, p0, U, flags)
    hidden = torch.from_numpy(network(model, x, hidden=True))
    w, b = model["layers"][-1]
    want = F.conv3d(torch.cat([hidden, torch.from_numpy(pS).double()], 1), torch.from_numpy(w).double(),
                    torch.from_numpy(b).double()).numpy() * sc
    assert np.abs(p - want).max() <= 1e-6 * np.abs(want).max()
