"""The CPU restatement of the input block of torch/lib/model.lua:27-150 and :357-387 (tests/inputs_oracle.py:
inputChannels, normalizeInput, normalizeInputFunc, normalizeInputChan, addPressureSkip) against an independent
float64 evaluation: the divergence, the scale and the channel join restated here in numpy, the convolutions in
torch.nn.functional.  This pins the semantics the GPU path is then compared with (tests/test_gpu_cnn_inputs.py)."""
import itertools

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import oracle
from fluidnet_b200 import synth
from inputs_oracle import model_forward_inputs
from test_oracle_model_graph import torch_stack

# Every inputChannels set the reference can build: flags on, and UDiv or div (tfluids.VelocityUpdate needs UDiv).
SETS = [dict(pDiv=p, UDiv=u, div=d, flags=True) for p, u, d in itertools.product([False, True], repeat=3) if u or d]


def set_id(ch):
    return "+".join(k for k in ("pDiv", "UDiv", "div") if ch[k])


def divergence64(U1, flags):
    """tfluids.VelocityDivergence on fluid cells off the border (tfluids/generic/tfluids.cu), in float64."""
    u = U1.astype(np.float64)
    is3d = U1.shape[1] == 3
    fl = flags[:, 0].astype(np.int32)
    d = np.zeros(fl.shape, np.float64)
    d[..., :-1] += u[:, 0, ..., :-1] - u[:, 0, ..., 1:]
    d[..., :-1, :] += u[:, 1, ..., :-1, :] - u[:, 1, ..., 1:, :]
    if is3d:
        d[:, :-1] += u[:, 2, :-1] - u[:, 2, 1:]
    inner = np.zeros(fl.shape, bool)
    if is3d:
        inner[:, 1:-1, 1:-1, 1:-1] = True
    else:
        inner[:, :, 1:-1, 1:-1] = True
    return np.where(inner & ((fl & 1) != 0), d, 0.0)[:, None]


def reference_p(model, pDiv, U1, flags, ch, normalize, func, chan, skip, threshold=1e-5):
    """p and the scale of lib/model.lua in float64 (occupancy: 0 fluid, 1 obstacle)."""
    div = divergence64(U1, flags)
    fields = {"UDiv": U1.astype(np.float64), "pDiv": pDiv.astype(np.float64), "div": div}
    b = pDiv.shape[0]
    scale = np.ones(b)
    if normalize:
        for ib in range(b):
            f = fields[chan][ib].ravel()
            s = f.std(ddof=1) if func == "std" else np.sqrt((f * f).sum())
            scale[ib] = max(s, threshold)
    sc = scale.reshape(b, 1, 1, 1, 1)
    occ = np.where(flags.astype(np.int32) & 1, 0.0, 1.0)
    parts = [(fields["pDiv"] / sc, ch["pDiv"]), (fields["UDiv"] / sc, ch["UDiv"]), (div / sc, ch["div"]), (occ, True)]
    x = np.concatenate([a for a, on in parts if on], axis=1)
    if not skip:
        return torch_stack(x, model) * (sc if normalize else 1.0), scale
    is3d = model["is3D"]
    t = torch.from_numpy(x)
    if not is3d:
        t = t[:, :, 0]
    nl = len(model["layers"])
    for li, (w, bias) in enumerate(model["layers"]):
        if li == nl - 1:                                       # JoinTable(2)({hl, pDiv}) (:357-361)
            ps = torch.from_numpy(fields["pDiv"] / sc)
            t = torch.cat([t, ps if is3d else ps[:, :, 0]], dim=1)
        wt, bt = torch.from_numpy(w).double(), torch.from_numpy(bias).double()
        t = F.conv3d(t, wt, bt, padding=w.shape[-1] // 2) if is3d else F.conv2d(t, wt[:, :, 0], bt,
                                                                                padding=w.shape[-1] // 2)
        if li < nl - 1:
            t = torch.sigmoid(t) if model.get("nonlinType") == "sigmoid" else F.relu(t)
    p = t.numpy() if is3d else t.numpy()[:, :, None]
    return p * (sc if normalize else 1.0), scale


def run_case(is3d, ch, normalize=True, func="std", chan="UDiv", skip=False, model_type="default"):
    orc = oracle.Oracle()
    n = 8 if is3d else 14
    flags = synth.make_flags(n, n + 2, n if is3d else 1, is3d, nb=2, geometry=False)
    U = synth.make_smooth_velocity(flags, is3d, amp=1.5)
    orc.setWallBcsForward(U, flags)
    p0 = (synth.make_density(flags, seed=5) - np.float32(0.5)) * np.float32(0.2)
    inputs = dict(inputChannels=ch, normalizeInput=normalize, normalizeInputFunc=func, normalizeInputChan=chan,
                  addPressureSkip=skip)
    model = synth.make_model(is3d, model_type=model_type, inputs=inputs)
    assert model["layers"][0][0].shape[1] == ch["pDiv"] + (3 if is3d else 2) * ch["UDiv"] + ch["div"] + 1
    assert model["layers"][-1][0].shape[1] == model["layers"][-2][0].shape[0] + skip
    p, U2, scale = model_forward_inputs(orc, model, p0, U, flags, **model["inputs"])
    U1 = U.copy()
    orc.setWallBcsForward(U1, flags, as_mask_multiply=True)
    want, want_scale = reference_p(model, p0, U1, flags, ch, normalize, func, chan, skip)
    assert np.abs(scale - want_scale).max() <= 1e-6 * want_scale.max(), (scale, want_scale)
    for b in range(2):
        assert np.abs(p[b] - want[b]).max() <= 2e-6 * max(np.abs(want[b]).max(), 1e-3)
    if not normalize:
        assert np.all(scale == 1.0)
        Uw = U1.copy()                                         # no ApplyScale around the velocity update
        orc.velocityUpdateForward(Uw, flags, p)
        orc.setWallBcsForward(Uw, flags, as_mask_multiply=True)
        assert np.array_equal(U2, Uw)


@pytest.mark.parametrize("ch", SETS, ids=set_id)
@pytest.mark.parametrize("is3d", [True, False], ids=["3d", "2d"])
def test_every_input_set(is3d, ch):
    run_case(is3d, ch, chan="div" if ch["div"] and not ch["UDiv"] else "UDiv")


@pytest.mark.parametrize("chan", ["UDiv", "pDiv", "div"])
@pytest.mark.parametrize("func", ["std", "norm"])
@pytest.mark.parametrize("is3d", [True, False], ids=["3d", "2d"])
def test_scale_function_and_channel(is3d, func, chan):
    run_case(is3d, dict(pDiv=True, UDiv=True, div=True, flags=True), func=func, chan=chan)


@pytest.mark.parametrize("ch", [SETS[-1], dict(pDiv=False, UDiv=True, div=False, flags=True)], ids=set_id)
@pytest.mark.parametrize("is3d", [True, False], ids=["3d", "2d"])
def test_normalization_off(is3d, ch):
    run_case(is3d, ch, normalize=False)


@pytest.mark.parametrize("model_type,ch", [("default", SETS[-1]), ("default", dict(pDiv=False, UDiv=True, div=False,
                                                                                      flags=True)),
                                           ("yang", dict(pDiv=True, UDiv=False, div=True, flags=True))],
                         ids=["default-all", "default-UDiv", "yang"])
@pytest.mark.parametrize("is3d", [True, False], ids=["3d", "2d"])
def test_pressure_skip(is3d, model_type, ch):
    run_case(is3d, ch, skip=True, model_type=model_type)


def test_defaults_are_the_default_graph():
    """No keywords and the explicit defaults give the bits of oracle.model_forward (the 'default' input block)."""
    orc = oracle.Oracle()
    flags = synth.make_flags(8, 8, 8, True, nb=2)
    U = synth.make_smooth_velocity(flags, True)
    p0 = (synth.make_density(flags, seed=5) - np.float32(0.5)) * np.float32(0.2)
    model = synth.make_model(True)
    want = oracle.model_forward(orc, model, p0, U, flags)
    a = model_forward_inputs(orc, model, p0, U, flags)
    b = model_forward_inputs(orc, model, p0, U, flags, inputChannels=dict(pDiv=True, UDiv=False, div=True, flags=True),
                             normalizeInput=True, normalizeInputFunc="std", normalizeInputChan="UDiv",
                             addPressureSkip=False)
    for x, y, z in zip(want, a, b):
        assert np.array_equal(x, y) and np.array_equal(x, z)
