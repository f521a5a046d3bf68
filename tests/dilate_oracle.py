"""The dilated-bank graph of torch/lib/model.lua:252-361 (banksType 'dilate') on the CPU, for the tests.

`model_forward_dilated` is tests/bank_oracle.model_forward_banked for a model whose banks have "type": 'dilate':
the same input normalisation and velocity update around the network, and a stage loop in the reference's order --
at banksSplitStage every bank takes the hidden layer as it is (model.lua:279-285), the stages in between run bank i's
convolution dilated by 2^(i-1) on every axis with padding 2^(i-1) (k-1)/2 (nn.{Spatial,Volumetric}DilatedConvolution,
lib/model_utils.lua:122-146), then its non-linearity and pooling, and at banksJoinStage the banks are concatenated
along the channels in bank order or summed left to right, without upsampling (model.lua:300-318).  Any other model
goes to model_forward_banked.

Bank 1's convolutions, and every convolution outside the banks, go through the oracle backend's `conv`, as in
bank_oracle; a dilated convolution is a float64 sum over its taps rounded once to float32.
tests/test_oracle_model_dilate.py pins it on torch.nn.functional.conv{2,3}d(dilation=d)."""
import numpy as np

from bank_oracle import _stage, model_forward_banked


def conv_dilated(x, w, b, is3d, d, relu=False):
    """x [B][cin][Z][Y][X] (float32) * w [cout][cin][kz][k][k] + b with dilation d on every axis (z only in 3-D) and
    zero padding d (k-1)/2, so the grid is kept: out[x] = sum_t w[t] in[x + (t - (k-1)/2) d].  Float64 sums."""
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
    out = acc.astype(np.float32)
    return np.maximum(out, 0) if relu else out


class _Dilated:
    """A stand-in for the oracle backend whose `conv` is dilated by d (the only backend call _stage makes)."""

    def __init__(self, d):
        self.d = d

    def conv(self, x, w, bias, is3d, relu=False):
        return conv_dilated(x, w, bias, is3d, self.d, relu)


def is_dilated(model):
    bk = model.get("banks")
    return bool(bk) and bk.get("type") == "dilate"


def network(be, model, x):
    """The convolution stages of a 'dilate' model on the network input x [b][c][z][y][x] -> p_net."""
    banks = model["banks"]
    n, s, j = banks["num"], banks["split_stage"], banks["join_stage"]
    hl = [x]
    for li, layer in enumerate(model["layers"]):
        lid = li + 1
        if n > 1 and lid == s:
            hl = [hl[0]] * n
        if n > 1 and lid == j:
            if banks["aggregate"] == "concat":
                hl = [np.ascontiguousarray(np.concatenate(hl, axis=1))]
            else:
                acc = hl[0]
                for h in hl[1:]:
                    acc = (acc + h).astype(np.float32)
                hl = [acc]
        convs = layer if isinstance(layer[0], (tuple, list)) else [layer]
        assert len(convs) == len(hl)
        hl = [_stage(be if i == 0 else _Dilated(2 ** i), model, li, w, b, h)
              for i, ((w, b), h) in enumerate(zip(convs, hl))]
    assert len(hl) == 1
    return hl[0]


def model_forward_dilated(be, model, pDiv, UDiv, flags, threshold=1e-5):
    """model_forward_banked with the 'dilate' bank semantics.  Returns (p, U, scale)."""
    if not is_dilated(model):
        return model_forward_banked(be, model, pDiv, UDiv, flags, threshold)
    U1 = UDiv.copy()
    be.setWallBcsForward(U1, flags, as_mask_multiply=True)
    div = be.velocityDivergenceForward(U1, flags)
    b = U1.shape[0]
    scales = np.empty(b, np.float32)
    for ib in range(b):
        scales[ib] = max(np.float32(be.sampleStd(U1[ib])), np.float32(threshold))
    sc = scales.reshape(b, 1, 1, 1, 1)
    pS = (pDiv / sc).astype(np.float32)
    US = (U1 / sc).astype(np.float32)
    divS = (div / sc).astype(np.float32)
    occ = be.flagsToOccupancy(flags)
    x = np.ascontiguousarray(np.concatenate([pS, divS, occ], axis=1))
    p = network(be, model, x)
    U2 = np.ascontiguousarray(US.copy())
    be.velocityUpdateForward(U2, flags, p)
    p = (p * sc).astype(np.float32)
    U2 = np.ascontiguousarray((U2 * sc).astype(np.float32))
    be.setWallBcsForward(U2, flags, as_mask_multiply=True)
    return p, U2, scales
