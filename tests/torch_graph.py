"""The projection network's stages restated on torch.nn.functional, which the oracle's graph, bank, dilation and
input-block semantics are pinned on."""
import torch
import torch.nn.functional as F


def torch_stage(t, model, li, w, b):
    is3d = model["is3D"]
    nl = len(model["layers"])
    pool = model.get("pool") or [1] * nl
    up = model.get("up") or [1] * nl
    wt, bt = torch.from_numpy(w).double(), torch.from_numpy(b).double()
    k = w.shape[-1]
    t = F.conv3d(t, wt, bt, padding=k // 2) if is3d else F.conv2d(t, wt[:, :, 0], bt, padding=k // 2)
    s = up[li]
    if s > 1:
        if is3d:
            bsz, ct, d, h, w_ = t.shape
            no = ct // s ** 3
            out = torch.empty(bsz, no, d * s, h * s, w_ * s, dtype=t.dtype)
            for st in range(s):
                for sh in range(s):
                    for sw in range(s):
                        out[:, :, st::s, sh::s, sw::s] = t[:, torch.arange(no) * s ** 3 + (st * s + sh) * s + sw]
            t = out
        else:
            t = F.pixel_shuffle(t, s)
    if li < nl - 1:
        t = torch.sigmoid(t) if model.get("nonlinType") == "sigmoid" else F.relu(t)
    if pool[li] > 1:
        t = (F.avg_pool3d if is3d else F.avg_pool2d)(t, pool[li])
    return t


def torch_stack(x, model):
    is3d = model["is3D"]
    nl = len(model["layers"])
    pool = model.get("pool") or [1] * nl
    up = model.get("up") or [1] * nl
    t = torch.from_numpy(x).double()
    if not is3d:
        t = t[:, :, 0]
    for li, (w, b) in enumerate(model["layers"]):
        wt, bt = torch.from_numpy(w).double(), torch.from_numpy(b).double()
        k = w.shape[-1]
        if is3d:
            t = F.conv3d(t, wt, bt, padding=k // 2)
        else:
            t = F.conv2d(t, wt[:, :, 0], bt, padding=k // 2)
        s = up[li]
        if s > 1:
            if is3d:                      # explicit index form of volumetric_convolution_upsample.lua
                bsz, ct, d, h, w_ = t.shape
                no = ct // s ** 3
                out = torch.empty(bsz, no, d * s, h * s, w_ * s, dtype=t.dtype)
                for st in range(s):
                    for sh in range(s):
                        for sw in range(s):
                            ch = torch.arange(no) * s ** 3 + (st * s + sh) * s + sw
                            out[:, :, st::s, sh::s, sw::s] = t[:, ch]
                t = out
            else:
                t = F.pixel_shuffle(t, s)
        if li < nl - 1:
            t = torch.sigmoid(t) if model.get("nonlinType") == "sigmoid" else F.relu(t)
        if pool[li] > 1:
            fn = {(True, "avg"): F.avg_pool3d, (True, "max"): F.max_pool3d, (False, "avg"): F.avg_pool2d,
                  (False, "max"): F.max_pool2d}[(is3d, model.get("poolType", "avg"))]
            t = fn(t, pool[li])
    if not is3d:
        t = t[:, :, None]
    return t.numpy()
