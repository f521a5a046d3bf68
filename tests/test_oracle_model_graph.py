"""The oracle's restatement of the single-bank model graphs of torch/lib/model.lua:164-340 ('default', 'tog',
'yang': convolution, ConvolutionUpsample pixel shuffle, non-linearity, pooling) against an independent
evaluation with torch.nn.functional in float64 -- the conv stack has no CPU source in the reference
(cudnn.torch), so this pins the graph semantics the GPU path is then compared with."""
import numpy as np
import pytest

import oracle
from fluidnet_b200 import synth
from torch_graph import torch_stack


@pytest.mark.parametrize("model_type", ["default", "tog", "yang"])
@pytest.mark.parametrize("is3d", [True, False])
def test_graph_matches_torch(is3d, model_type):
    orc = oracle.Oracle()
    n = 8 if is3d else 16
    flags = synth.make_flags(n, n, n if is3d else 1, is3d, nb=2, geometry=False)
    U = synth.make_smooth_velocity(flags, is3d, amp=1.0)
    orc.setWallBcsForward(U, flags)
    model = synth.make_model(is3d, model_type=model_type)
    if model_type == "tog":
        model["poolType"] = "max" if is3d else "avg"                   # cover both pooling types
    p0 = (synth.make_density(flags, seed=5) - np.float32(0.5)) * np.float32(0.1)
    p, U2, scale = oracle.model_forward(orc, model, p0, U, flags)
    # rebuild the network input exactly as model_forward does and push it through torch
    U1 = U.copy()
    orc.setWallBcsForward(U1, flags, as_mask_multiply=True)
    sc = scale.reshape(-1, 1, 1, 1, 1)
    x = np.concatenate([(p0 / sc).astype(np.float32), (orc.velocityDivergenceForward(U1, flags) / sc).astype(np.float32),
                        orc.flagsToOccupancy(flags)], axis=1)
    want = torch_stack(np.ascontiguousarray(x), model) * sc
    assert p.shape == flags.shape
    assert np.abs(p - want).max() <= 2e-6 * max(np.abs(want).max(), 1e-3)
