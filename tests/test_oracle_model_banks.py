"""The CPU restatement of the multi-resolution bank graph (oracle/model.py, lib/model.lua:252-361) against an
independent float64 evaluation with torch.nn.functional: avg_pool for the pyramid, interpolate(mode='nearest') for
the join's upsampling, cat / + for the aggregation.  The GPU path is then compared with the restatement."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import oracle
from fluidnet_b200 import synth
from torch_graph import torch_stage


def torch_banked(x, model):
    is3d = model["is3D"]
    bk = model["banks"]
    n, s, j = bk["num"], bk["split_stage"], bk["join_stage"]
    t = torch.from_numpy(x).double()
    if not is3d:
        t = t[:, :, 0]
    hl = [t]
    for li, layer in enumerate(model["layers"]):
        if li + 1 == s:
            for i in range(1, n):
                hl.append((F.avg_pool3d if is3d else F.avg_pool2d)(hl[-1], 2))
        if li + 1 == j:
            ups = [hl[0]] + [F.interpolate(h, scale_factor=2 ** i, mode="nearest") for i, h in enumerate(hl) if i > 0]
            hl = [torch.cat(ups, dim=1)] if bk["aggregate"] == "concat" else [sum(ups[1:], ups[0])]
        convs = layer if isinstance(layer, list) else [layer]
        hl = [torch_stage(h, model, li, w, b) for (w, b), h in zip(convs, hl)]
    t = hl[0]
    if not is3d:
        t = t[:, :, None]
    return t.numpy()


# (is3d, model_type, num, aggregate, split, join, grid)
CASES = {
    "3d-n2-concat": (True, "default", 2, "concat", 1, 3, (8, 8, 8)),
    "3d-n3-concat": (True, "default", 3, "concat", 1, 3, (8, 12, 16)),
    "3d-n2-add": (True, "default", 2, "add", 1, 3, (8, 8, 12)),
    "3d-n3-add": (True, "default", 3, "add", 1, 3, (12, 8, 8)),
    "3d-n2-s2j4-concat": (True, "default", 2, "concat", 2, 4, (6, 8, 10)),
    "2d-n2-concat": (False, "default", 2, "concat", 1, 3, (1, 16, 12)),
    "2d-n3-concat": (False, "default", 3, "concat", 1, 3, (1, 16, 20)),
    "2d-n2-add": (False, "default", 2, "add", 1, 3, (1, 12, 16)),
    "2d-n3-add": (False, "default", 3, "add", 1, 3, (1, 16, 16)),
    "2d-n2-s2j4-add": (False, "default", 2, "add", 2, 4, (1, 10, 14)),
    "2d-tog-n2-concat": (False, "tog", 2, "concat", 1, 3, (1, 16, 16)),
}


@pytest.mark.parametrize("case", list(CASES))
def test_banked_graph_matches_torch(case):
    is3d, model_type, num, agg, s, j, (nz, ny, nx) = CASES[case]
    orc = oracle.Oracle()
    flags = synth.make_flags(nx, ny, nz, is3d, nb=2, geometry=False)
    U = synth.make_smooth_velocity(flags, is3d, amp=1.0)
    orc.setWallBcsForward(U, flags)
    model = synth.make_model(is3d, model_type=model_type,
                             banks={"num": num, "split_stage": s, "join_stage": j, "aggregate": agg})
    p0 = (synth.make_density(flags, seed=5) - np.float32(0.5)) * np.float32(0.1)
    p, U2, scale = oracle.model_forward(orc, model, p0, U, flags)
    U1 = U.copy()
    orc.setWallBcsForward(U1, flags, as_mask_multiply=True)
    sc = scale.reshape(-1, 1, 1, 1, 1)
    x = np.concatenate([(p0 / sc).astype(np.float32), (orc.velocityDivergenceForward(U1, flags) / sc).astype(np.float32),
                        orc.flagsToOccupancy(flags)], axis=1)
    want = torch_banked(np.ascontiguousarray(x), model) * sc
    assert p.shape == flags.shape
    assert np.abs(p - want).max() <= 2e-6 * max(np.abs(want).max(), 1e-3)


def test_single_bank_is_the_plain_graph():
    """num = 1 draws the same weights as no banks, and the 1-bank graph then computes the plain graph's bits."""
    orc = oracle.Oracle()
    flags = synth.make_flags(8, 8, 8, True, nb=1, geometry=False)
    U = synth.make_smooth_velocity(flags, True, amp=1.0)
    orc.setWallBcsForward(U, flags)
    plain = synth.make_model(True)
    one = synth.make_model(True, banks={"num": 1, "split_stage": 1, "join_stage": 3, "aggregate": "concat"})
    for (w0, b0), (w1, b1) in zip(plain["layers"], one["layers"]):
        assert np.array_equal(w0, w1) and np.array_equal(b0, b1)
    p0 = np.zeros_like(flags)
    a = oracle.model_forward(orc, plain, p0, U, flags)
    b = oracle.model_forward(orc, one, p0, U, flags)
    for u, v in zip(a, b):
        assert np.array_equal(u, v)
