"""The multi-resolution bank graph of torch/lib/model.lua:252-361 (banksType 'mres') on the CPU, for the tests.

`model_forward_banked` is oracle.model_forward with banks: the same input normalisation and velocity update
around the network, and a stage loop that follows the reference's order -- before banksSplitStage the hidden
layer is split into a pyramid (bank i = 2x average pool of bank i-1), the stages in between run one
convolution (+ pixel shuffle, non-linearity, pooling) per bank, and before banksJoinStage bank i is upsampled
nearest by 2^(i-1) and the banks are concatenated along the channels in bank order (nn.JoinTable) or summed left
to right (nn.CAddTable).  Without "banks" in the model it returns what oracle.model_forward returns.  The
convolutions go through the oracle backend's `conv`; everything else is numpy in float32 (float64 sums for the
average pools).  tests/test_oracle_model_banks.py pins it on torch.nn.functional."""
import numpy as np

import oracle


def _avg_pool(x, q, is3d):
    b_, c_, z_, y_, x_ = x.shape
    qz = q if is3d else 1
    v = x.reshape(b_, c_, z_ // qz, qz, y_ // q, q, x_ // q, q)
    return (v.astype(np.float64).sum(axis=(3, 5, 7)) / (qz * q * q)).astype(np.float32)


def _upsample(x, r, is3d):
    x = np.repeat(np.repeat(x, r, axis=3), r, axis=4)
    return np.repeat(x, r, axis=2) if is3d else x


def _stage(be, model, li, w, bias, x):
    """One convolution stage of model.lua:320-357 (as in oracle.model_forward)."""
    is3d = model["is3D"]
    nl = len(model["layers"])
    pool = model.get("pool") or [1] * nl
    up = model.get("up") or [1] * nl
    sigmoid = model.get("nonlinType", "relu") == "sigmoid"
    plain = up[li] == 1 and pool[li] == 1 and not sigmoid
    x = be.conv(x, w, bias, is3d, relu=(plain and li < nl - 1))
    if plain:
        return x
    if up[li] > 1:
        s_ = up[li]
        b_, ct, z_, y_, x_ = x.shape
        if is3d:
            no = ct // s_ ** 3
            x = x.reshape(b_, no, s_, s_, s_, z_, y_, x_).transpose(0, 1, 5, 2, 6, 3, 7, 4)
            x = np.ascontiguousarray(x).reshape(b_, no, z_ * s_, y_ * s_, x_ * s_)
        else:
            no = ct // s_ ** 2
            x = x.reshape(b_, no, s_, s_, z_, y_, x_).transpose(0, 1, 4, 5, 2, 6, 3)
            x = np.ascontiguousarray(x).reshape(b_, no, z_, y_ * s_, x_ * s_)
    if li < nl - 1:
        x = (1.0 / (1.0 + np.exp(-x.astype(np.float64)))).astype(np.float32) if sigmoid else np.maximum(x, 0)
    if pool[li] > 1:
        q = pool[li]
        if model.get("poolType", "avg") == "max":
            b_, c_, z_, y_, x_ = x.shape
            qz = q if is3d else 1
            x = x.reshape(b_, c_, z_ // qz, qz, y_ // q, q, x_ // q, q).max(axis=(3, 5, 7))
        else:
            x = _avg_pool(x, q, is3d)
    return np.ascontiguousarray(x, np.float32)


def network(be, model, x):
    """The convolution stages on the network input x [b][3][z][y][x] -> p_net."""
    is3d = model["is3D"]
    banks = model.get("banks")
    n = banks["num"] if banks else 1
    s, j = (banks["split_stage"], banks["join_stage"]) if banks else (0, 0)
    hl = [x]
    for li, layer in enumerate(model["layers"]):
        lid = li + 1
        if n > 1 and lid == s:
            for i in range(1, n):
                hl.append(_avg_pool(hl[i - 1], 2, is3d))
        if n > 1 and lid == j:
            ups = [hl[0]] + [_upsample(hl[i], 2 ** i, is3d) for i in range(1, n)]
            if banks["aggregate"] == "concat":
                hl = [np.ascontiguousarray(np.concatenate(ups, axis=1))]
            else:
                acc = ups[0]
                for u in ups[1:]:
                    acc = (acc + u).astype(np.float32)
                hl = [acc]
        convs = layer if isinstance(layer[0], (tuple, list)) else [layer]
        assert len(convs) == len(hl)
        hl = [_stage(be, model, li, w, b, h) for (w, b), h in zip(convs, hl)]
    assert len(hl) == 1
    return hl[0]


def model_forward_banked(be, model, pDiv, UDiv, flags, threshold=1e-5):
    """oracle.model_forward with the bank semantics of lib/model.lua:252-361.  Returns (p, U, scale)."""
    if not model.get("banks"):
        return oracle.model_forward(be, model, pDiv, UDiv, flags, threshold)
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
