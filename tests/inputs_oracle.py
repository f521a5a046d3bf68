"""The input block of torch/lib/model.lua:27-150 and :357-387 on the CPU, for the tests: the mconf keys
inputChannels, normalizeInput, normalizeInputFunc, normalizeInputChan and addPressureSkip around the network.

`model_forward_inputs` is oracle.model_forward with that block, the network itself run by tests/bank_oracle.py's
stage loop (single-bank and banked graphs alike); with the default keywords it computes what oracle.model_forward
computes.  The operators go through the oracle backend; the scale is taken from float64 sums as for 'std'.
tests/test_oracle_model_inputs.py pins it on a float64 numpy / torch.nn.functional evaluation."""
import numpy as np

from bank_oracle import network

DEFAULT_CHANNELS = {"pDiv": True, "UDiv": False, "div": True, "flags": True}      # lib/default_conf.lua:76-81


def model_input(be, pDiv, UDiv, flags, threshold=1e-5, inputChannels=None, normalizeInput=True,
                normalizeInputFunc="std", normalizeInputChan="UDiv"):
    """The network input x (nn.JoinTable(2) of the selected channels in the order pDiv, UDiv, div, occupancy), the
    scaled pDiv and UDiv, and the scale.  Returns (x, pS, US, sc [b,1,1,1,1], scales [b])."""
    ch = dict(DEFAULT_CHANNELS, **(inputChannels or {}))
    U1 = UDiv.copy()
    be.setWallBcsForward(U1, flags, as_mask_multiply=True)              # model.lua:81-84
    div = be.velocityDivergenceForward(U1, flags)                       # :86-89
    b = U1.shape[0]
    scales = np.ones(b, np.float32)                                     # no scale node without normalizeInput (:92)
    if normalizeInput:                                                  # :92-117
        field = {"UDiv": U1, "pDiv": pDiv, "div": div}[normalizeInputChan]                   # :108-116
        for ib in range(b):
            if normalizeInputFunc == "std":                             # nn.StandardDeviation (:96-97)
                s = np.float32(be.sampleStd(field[ib]))
            else:                                                       # Power(2), Sum, Sqrt (:98-102)
                f = np.asarray(field[ib], np.float32)
                s = np.float32(np.sqrt(np.sum((f * f).astype(np.float64))))
            scales[ib] = max(s, np.float32(threshold))                  # nn.Clamp (:106)
    sc = scales.reshape(b, 1, 1, 1, 1)
    if normalizeInput:                                                  # :119-130 (ApplyScale)
        pS = (pDiv / sc).astype(np.float32)
        US = (U1 / sc).astype(np.float32)
        divS = (div / sc).astype(np.float32)
    else:
        pS, US, divS = np.asarray(pDiv, np.float32), U1, div
    occ = be.flagsToOccupancy(flags)                                    # :144-147
    chans = [c for c, on in ((pS, ch["pDiv"]), (US, ch["UDiv"]), (divS, ch["div"]), (occ, ch["flags"])) if on]
    x = np.ascontiguousarray(np.concatenate(chans, axis=1))             # :133-150
    return x, pS, US, sc, scales


def model_forward_inputs(be, model, pDiv, UDiv, flags, threshold=1e-5, inputChannels=None, normalizeInput=True,
                         normalizeInputFunc="std", normalizeInputChan="UDiv", addPressureSkip=False):
    """lib/model.lua:27-401 with the input block.  model as for bank_oracle.network.  Returns (p, U, scale)."""
    x, pS, US, sc, scales = model_input(be, pDiv, UDiv, flags, threshold, inputChannels, normalizeInput,
                                        normalizeInputFunc, normalizeInputChan)
    if addPressureSkip:                                                 # :357-361 JoinTable(2)({hl, pDiv})
        # The hidden layer before the last convolution: the stage loop with an exact 1x1 identity in place of the
        # last convolution (x * 1 + 0 * y + 0 is exact), then the last convolution on [hidden, pDiv].
        w, b = model["layers"][-1]
        c = w.shape[1] - 1
        ident = np.zeros((c, c) + w.shape[2:], np.float32)
        ident[np.arange(c), np.arange(c)] = 1.0
        hidden = network(be, dict(model, layers=model["layers"][:-1] + [(ident, np.zeros(c, np.float32))]), x)
        p = be.conv(np.ascontiguousarray(np.concatenate([hidden, pS], axis=1)), w, b, model["is3D"], relu=False)
    else:
        p = network(be, model, x)
    U2 = np.ascontiguousarray(US.copy())
    be.velocityUpdateForward(U2, flags, p)                              # :380
    if normalizeInput:
        p = (p * sc).astype(np.float32)                                 # :384-387
        U2 = np.ascontiguousarray((U2 * sc).astype(np.float32))
    be.setWallBcsForward(U2, flags, as_mask_multiply=True)              # :390
    return p, U2, scales


def model_forward_of_model(be, model, pDiv, UDiv, flags, threshold=1e-5):
    """oracle.model_forward's signature with the block read from model["inputs"] (synth.make_model(inputs=)), so that
    oracle.simulate can run such a model."""
    return model_forward_inputs(be, model, pDiv, UDiv, flags, threshold, **(model.get("inputs") or {}))
