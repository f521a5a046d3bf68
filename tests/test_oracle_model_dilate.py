"""The CPU restatement of the dilated-bank graph (tests/dilate_oracle.py, banksType 'dilate', lib/model.lua:252-361)
against an independent float64 evaluation with torch.nn.functional: conv{2,3}d(dilation=2^(i-1), padding
2^(i-1) (k-1)/2) for bank i, cat / + for the aggregation, no upsampling.  The GPU path is then compared with the
restatement.  Grids are chosen not divisible by the dilations, and some have an axis shorter than the largest one."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import oracle
from dilate_oracle import conv_dilated, model_forward_dilated
from fluidnet_b200 import synth
from test_oracle_model_banks import torch_stage


def torch_stage_dilated(t, model, li, w, b, d):
    """torch_stage with the convolution dilated by d (dilated stages have no upsampling, model_utils.lua:125)."""
    if d == 1:
        return torch_stage(t, model, li, w, b)
    is3d = model["is3D"]
    nl = len(model["layers"])
    pool = model.get("pool") or [1] * nl
    wt, bt = torch.from_numpy(w).double(), torch.from_numpy(b).double()
    pad = d * (w.shape[-1] - 1) // 2
    t = F.conv3d(t, wt, bt, padding=pad, dilation=d) if is3d else F.conv2d(t, wt[:, :, 0], bt, padding=pad, dilation=d)
    if li < nl - 1:
        t = torch.sigmoid(t) if model.get("nonlinType") == "sigmoid" else F.relu(t)
    if pool[li] > 1:
        t = (F.avg_pool3d if is3d else F.avg_pool2d)(t, pool[li])
    return t


def torch_dilated(x, model):
    is3d = model["is3D"]
    bk = model["banks"]
    n, s, j = bk["num"], bk["split_stage"], bk["join_stage"]
    t = torch.from_numpy(x).double()
    if not is3d:
        t = t[:, :, 0]
    hl = [t]
    for li, layer in enumerate(model["layers"]):
        if li + 1 == s:
            hl = hl * n
        if li + 1 == j:
            hl = [torch.cat(hl, dim=1)] if bk["aggregate"] == "concat" else [sum(hl[1:], hl[0])]
        convs = layer if isinstance(layer, list) else [layer]
        hl = [torch_stage_dilated(h, model, li, w, b, 2 ** i) for i, ((w, b), h) in enumerate(zip(convs, hl))]
    t = hl[0]
    if not is3d:
        t = t[:, :, None]
    return t.numpy()


def dilate(num, agg, s=1, j=3):
    return {"num": num, "split_stage": s, "join_stage": j, "aggregate": agg, "type": "dilate"}


# (is3d, model_type, banks, (nz, ny, nx)).  The dilations 2^(N-1) divide no axis of the 'default' grids; the N = 4
# cases have dilation 8 above some axis, so its taps fall outside the grid on both sides.
CASES = {
    "3d-n2-concat": (True, "default", dilate(2, "concat"), (5, 7, 9)),
    "3d-n3-concat": (True, "default", dilate(3, "concat"), (6, 5, 11)),
    "3d-n2-add": (True, "default", dilate(2, "add"), (7, 6, 5)),
    "3d-n4-add": (True, "default", dilate(4, "add"), (5, 9, 7)),
    "3d-n4-concat-d8-over-axes": (True, "default", dilate(4, "concat"), (3, 6, 7)),
    "3d-n3-s2j4-concat": (True, "default", dilate(3, "concat", 2, 4), (5, 6, 9)),
    "3d-yang-n3-add": (True, "yang", dilate(3, "add", 1, 2), (5, 6, 7)),
    "3d-tog-n2-add": (True, "tog", dilate(2, "add"), (8, 12, 12)),
    "3d-tog-n2-concat": (True, "tog", dilate(2, "concat"), (8, 8, 12)),
    "2d-n2-concat": (False, "default", dilate(2, "concat"), (1, 13, 11)),
    "2d-n3-add": (False, "default", dilate(3, "add"), (1, 9, 15)),
    "2d-n4-concat": (False, "default", dilate(4, "concat"), (1, 7, 10)),
    "2d-n2-s2j4-add": (False, "default", dilate(2, "add", 2, 4), (1, 10, 13)),
    "2d-yang-n2-concat-s2j3": (False, "yang", dilate(2, "concat", 2, 3), (1, 12, 9)),
    "2d-tog-n3-concat": (False, "tog", dilate(3, "concat"), (1, 18, 22)),
}


def network_input(orc, model, flags, U, p0, scale):
    U1 = U.copy()
    orc.setWallBcsForward(U1, flags, as_mask_multiply=True)
    sc = scale.reshape(-1, 1, 1, 1, 1)
    x = np.concatenate([(p0 / sc).astype(np.float32), (orc.velocityDivergenceForward(U1, flags) / sc).astype(np.float32),
                        orc.flagsToOccupancy(flags)], axis=1)
    return np.ascontiguousarray(x), sc


@pytest.mark.parametrize("case", list(CASES))
def test_dilated_graph_matches_torch(case):
    is3d, model_type, bk, (nz, ny, nx) = CASES[case]
    orc = oracle.Oracle()
    flags = synth.make_flags(nx, ny, nz, is3d, nb=2, geometry=False)
    U = synth.make_smooth_velocity(flags, is3d, amp=1.0)
    orc.setWallBcsForward(U, flags)
    model = synth.make_model(is3d, model_type=model_type, banks=bk)
    assert model["banks"]["type"] == "dilate"
    p0 = (synth.make_density(flags, seed=5) - np.float32(0.5)) * np.float32(0.1)
    p, U2, scale = model_forward_dilated(orc, model, p0, U, flags)
    x, sc = network_input(orc, model, flags, U, p0, scale)
    want = torch_dilated(x, model) * sc
    assert p.shape == flags.shape
    assert np.abs(p - want).max() <= 2e-6 * max(np.abs(want).max(), 1e-3)


@pytest.mark.parametrize("is3d", [True, False], ids=["3d", "2d"])
@pytest.mark.parametrize("d", [1, 2, 4, 8])
def test_dilated_convolution_matches_torch(is3d, d):
    """conv_dilated alone, on a grid with an axis shorter than d and axes d does not divide."""
    rs = np.random.RandomState(d)
    shape = (2, 3) + ((5, 7, 9) if is3d else (1, 7, 9))
    kz = 3 if is3d else 1
    x = rs.uniform(-1, 1, shape).astype(np.float32)
    w = rs.uniform(-1, 1, (4, 3, kz, 3, 3)).astype(np.float32)
    b = rs.uniform(-1, 1, 4).astype(np.float32)
    got = conv_dilated(x, w, b, is3d, d)
    xt, wt, bt = (torch.from_numpy(a).double() for a in (x, w, b))
    if is3d:
        want = F.conv3d(xt, wt, bt, padding=d, dilation=d).numpy()
    else:
        want = F.conv2d(xt[:, :, 0], wt[:, :, 0], bt, padding=d, dilation=d).numpy()[:, :, None]
    assert got.shape == want.shape
    assert np.abs(got - want).max() <= 1e-6 * np.abs(want).max()


def test_one_dilated_bank_is_the_plain_graph():
    """num = 1 'dilate' draws the same weights as no banks, and the restatement then equals oracle.model_forward."""
    orc = oracle.Oracle()
    flags = synth.make_flags(8, 8, 8, True, nb=1, geometry=False)
    U = synth.make_smooth_velocity(flags, True, amp=1.0)
    orc.setWallBcsForward(U, flags)
    plain = synth.make_model(True)
    one = synth.make_model(True, banks=dilate(1, "concat"))
    for (w0, b0), (w1, b1) in zip(plain["layers"], one["layers"]):
        assert np.array_equal(w0, w1) and np.array_equal(b0, b1)
    p0 = np.zeros_like(flags)
    a = oracle.model_forward(orc, plain, p0, U, flags)
    b = model_forward_dilated(orc, one, p0, U, flags)
    for u, v in zip(a, b):
        assert np.array_equal(u, v)


def test_dilate_and_mres_draw_the_same_weights():
    """synth.make_model gives 'dilate' the weight shapes (and values) of 'mres'; the restatements differ."""
    mres = synth.make_model(True, banks={"num": 2, "split_stage": 1, "join_stage": 3, "aggregate": "concat"})
    dil = synth.make_model(True, banks=dilate(2, "concat"))
    for a, b in zip(mres["layers"], dil["layers"]):
        a = a if isinstance(a, list) else [a]
        b = b if isinstance(b, list) else [b]
        for (wa, ba), (wb, bb) in zip(a, b):
            assert np.array_equal(wa, wb) and np.array_equal(ba, bb)
