"""Pressure-projection model (forward only) -- mirror of torch/lib/model.lua.

`ProjectionModel` plays the role of the nngraph module built by torch.defineModelGraph
(lib/model.lua:27-401), input block included (inputChannels, normalizeInput*, addPressureSkip):
`forward({pDiv, UDiv, flags})` returns `{p, U}` (lib/model.lua:421-450).  The whole graph runs inside libtfl.so
(tfl_cnn_project); weights are plain float32 arrays in Torch layout [cout][cin][kz][ky][kx].
"""
import ctypes as C

import numpy as np
import torch

from . import _lib, tfluids
from ._lib import TflError


DEFAULT_INPUTS = {"pDiv": True, "UDiv": False, "div": True, "flags": True}
NORM_FUNCS = {"std": 0, "norm": 1}
NORM_CHANS = {"UDiv": 0, "pDiv": 1, "div": 2}


def input_channel_count(inputChannels, is3D):
    """cin[0] of the network for an inputChannels table (lib/model.lua:28-46): pDiv, UDiv (2 or 3), div, flags."""
    ch = dict(DEFAULT_INPUTS, **(inputChannels or {}))
    return (1 if ch["pDiv"] else 0) + ((3 if is3D else 2) if ch["UDiv"] else 0) + (1 if ch["div"] else 0) + \
        (1 if ch["flags"] else 0)


def default_layers(is3D):
    """(cin, cout, k) of the 'default' modelType (lib/model.lua:179-186 2-D, :219-226 3-D)."""
    if is3D:
        return [(3, 8, 3), (8, 8, 3), (8, 8, 3), (8, 8, 1), (8, 1, 1)]
    return [(3, 16, 3), (16, 16, 3), (16, 16, 3), (16, 16, 3), (16, 1, 1)]


class ProjectionModel:
    def __init__(self, layers, is3D, device=None, normalizeInputThreshold=1e-5, pool=None, up=None,
                 poolType="avg", nonlinType="relu", banks=None, inputChannels=None, normalizeInput=True,
                 normalizeInputFunc="std", normalizeInputChan="UDiv", addPressureSkip=False, batchNorm=None):
        """layers: [(weight ndarray [cout * up^d][cin][kz][ky][kx], bias ndarray [cout * up^d]), ...]
        pool / up: per-layer pooling and ConvolutionUpsample sizes of the 'tog' graph (lib/model.lua:164-226),
        None = all 1 ('default', 'yang'); poolType 'avg' | 'max'; nonlinType 'relu' | 'sigmoid' | 'relu6'.
        banks: banks of convolutions (lib/model.lua:252-361), {"num": banksNum, "split_stage": banksSplitStage,
        "join_stage": banksJoinStage, "aggregate": 'concat' | 'add', "type": 'mres' | 'dilate'} (stages numbered
        from 1; a missing "type" is banksType 'mres', multi-resolution banks; 'dilate' dilates bank i's convolutions by
        2^(i-1) at full resolution); layers[l] of a banked stage (split_stage <= l + 1 < join_stage) is then a list of
        num (weight, bias) pairs, bank 1 first.  None: a single bank.
        inputChannels ({"pDiv", "UDiv", "div", "flags"} -> bool, missing keys at their defaults pDiv, div, flags),
        normalizeInput, normalizeInputFunc ('std' | 'norm'), normalizeInputChan ('UDiv' | 'pDiv' | 'div') and
        addPressureSkip are the mconf keys of lib/model.lua:27-150, :357-387; layers[0] takes the selected channels and
        with the skip the last layer takes one more, pDiv.  The library refuses what the reference cannot build.
        batchNorm: addBatchNorm (lib/model.lua:343-350), {"train": bool, "layers": [...]}: "layers" mirrors
        layers[:-1] (a banked stage holds a list with one entry per bank), each entry {"weight", "bias" (None for a
        module without batchNormAffine), "running_mean", "running_var", "eps"}.  train = True (the saved module's
        `train` field, true unless the model was put in evaluate mode) normalises with the statistics of the batch,
        False with the running statistics.  Such models run on the fp32 path, as do 'relu6' models."""
        ch = dict(DEFAULT_INPUTS, **(inputChannels or {}))
        if not ch["flags"]:
            raise TflError("Are you sure you dont want flags on input?")          # lib/model.lua:39-43
        if normalizeInputFunc not in NORM_FUNCS:
            raise TflError("Incorrect normalize input function")                  # :103
        if normalizeInputChan not in NORM_CHANS:
            raise TflError("Incorrect normalize input channel.")                  # :114
        cin_ = _lib.CnnInputs(int(bool(ch["pDiv"])), int(bool(ch["UDiv"])), int(bool(ch["div"])), int(bool(normalizeInput)),
                              NORM_FUNCS[normalizeInputFunc], NORM_CHANS[normalizeInputChan], int(bool(addPressureSkip)))
        self.is3D = bool(is3D)
        self.threshold = float(normalizeInputThreshold)
        self.ctx = tfluids.context(device)
        n = len(layers)
        pool = [1] * n if pool is None else [int(v) for v in pool]
        up = [1] * n if up is None else [int(v) for v in up]
        assert len(pool) == n and len(up) == n
        assert poolType in ("avg", "max") and nonlinType in ("relu", "sigmoid", "relu6")
        self.banks = dict(banks) if banks is not None else None
        if banks is not None:
            assert banks["aggregate"] in ("concat", "add"), "banksAggregateMethod must be 'concat' or 'add'"
            assert banks.get("type", "mres") in ("mres", "dilate"), "banksType must be 'mres' or 'dilate'"
        self._keep = []
        cin = (C.c_int32 * n)()
        cout = (C.c_int32 * n)()
        ks = (C.c_int32 * n)()
        cpool = (C.c_int32 * n)(*pool)
        cup = (C.c_int32 * n)(*up)
        # An invalid banks table is left to the library, which refuses it before it reads any weight.
        banks_ok = banks is not None and banks["num"] >= 1 and 1 <= banks["split_stage"] < banks["join_stage"] < n
        convs = []          # (w, b) stage by stage, bank 1 .. num for a banked stage
        for l, layer in enumerate(layers):
            per_bank = list(layer) if isinstance(layer[0], (tuple, list)) else [layer]
            if banks_ok and banks["num"] > 1 and banks["split_stage"] <= l + 1 < banks["join_stage"]:
                assert len(per_bank) == banks["num"], "stage %d needs one (weight, bias) per bank" % (l + 1)
            elif banks is None or banks_ok:
                assert len(per_bank) == 1, "stage %d is not banked" % (l + 1)
            for bk, (w, b) in enumerate(per_bank):
                w = np.ascontiguousarray(w, dtype=np.float32)
                b = np.ascontiguousarray(b, dtype=np.float32)
                assert w.ndim == 5 and b.ndim == 1 and b.shape[0] == w.shape[0]
                assert w.shape[3] == w.shape[4] and w.shape[2] == (w.shape[4] if is3D else 1)
                fan = up[l] ** (3 if is3D else 2)
                assert w.shape[0] % fan == 0, "ConvolutionUpsample layer: cout must be a multiple of up^d"
                shape = (w.shape[0] // fan, w.shape[1], w.shape[4])
                if bk == 0:
                    cout[l], cin[l], ks[l] = shape
                else:
                    assert shape == (cout[l], cin[l], ks[l]), "the banks of stage %d differ in shape" % (l + 1)
                convs.append((w, b))
        nc = len(convs)
        wp = (C.POINTER(C.c_float) * nc)()
        bp = (C.POINTER(C.c_float) * nc)()
        for i, (w, b) in enumerate(convs):
            self._keep += [w, b]
            wp[i] = w.ctypes.data_as(C.POINTER(C.c_float))
            bp[i] = b.ctypes.data_as(C.POINTER(C.c_float))
        norm = None
        if nonlinType == "relu6" or batchNorm is not None:
            norm = _lib.CnnNorm(int(nonlinType == "relu6"), int(batchNorm is not None),
                                int(bool(batchNorm is not None and batchNorm["train"])), None, None)
        if batchNorm is not None:
            entries = []        # conv order, as `convs` (the last convolution has no BN)
            assert len(batchNorm["layers"]) == n - 1, "batchNorm['layers'] mirrors layers[:-1]"
            for l, e in enumerate(batchNorm["layers"]):
                per_bank = list(e) if isinstance(e, (tuple, list)) else [e]
                fan = up[l] ** (3 if is3D else 2)
                nconv = len(layers[l]) if isinstance(layers[l][0], (tuple, list)) else 1
                assert len(per_bank) == nconv, "stage %d: one batch normalization per bank" % (l + 1)
                for bk in per_bank:
                    c = np.asarray(bk["running_mean"]).shape[0]
                    w = np.ones(c, np.float32) if bk.get("weight") is None else bk["weight"]
                    b = np.zeros(c, np.float32) if bk.get("bias") is None else bk["bias"]
                    arr = np.ascontiguousarray(np.stack([np.asarray(v, np.float32).reshape(c) for v in
                                                         (w, b, bk["running_mean"], bk["running_var"])]))
                    assert c * fan == convs[len(entries)][0].shape[0], \
                        "stage %d: batch normalization over %d channels, the stage has %d" % (l + 1, c, cout[l])
                    entries.append((arr, float(bk["eps"])))
            bnp = (C.POINTER(C.c_float) * len(entries))()
            eps = (C.c_float * len(entries))(*[e for _, e in entries])
            for i, (arr, _) in enumerate(entries):
                self._keep.append(arr)
                bnp[i] = arr.ctypes.data_as(C.POINTER(C.c_float))
            self._keep += [bnp, eps]
            norm.bn = bnp
            norm.eps = eps
        h = C.c_void_p()
        args = (self.ctx.h, 1 if is3D else 0, n, cin, cout, ks, cpool, cup, 1 if poolType == "max" else 0,
                1 if nonlinType == "sigmoid" else 0)
        cb = None
        if banks is not None:
            cb = _lib.CnnBanksEx(int(banks["num"]), int(banks["split_stage"]), int(banks["join_stage"]),
                                 1 if banks["aggregate"] == "add" else 0, 1 if banks.get("type") == "dilate" else 0)
        self.ctx.check(self.ctx.lib.tfl_cnn_create_model_norm(*args, C.byref(cb) if cb is not None else None,
                                                              C.byref(cin_), C.byref(norm) if norm is not None else None,
                                                              wp, bp, C.byref(h)))
        self.h = h
        self.last_scale = None

    @classmethod
    def from_reference_file(cls, model_path, mconf_path=None, device=None):
        """A model saved by the reference (torch/lib/save_model.lua: Torch7 binary network + `_mconf.bin`),
        read without Torch7 (fluidnet_b200/torch7.py).  Returns (model, mconf).
        The graph follows the mconf (modelType, nonlinType, poolType, the bank keys, the input block), each
        convolution goes to the (bank, stage) of its nngraph annotation, and the shapes are checked against the
        architecture.  Options and modules the library does not compute raise ValueError naming them."""
        from . import torch7
        ref = torch7.load_reference_model(model_path, mconf_path)
        bn = torch7.batch_norm_layers(ref["model"]) if ref["mconf"].get("addBatchNorm") else None
        opts = torch7.model_options(ref["mconf"], inputs=True, dilate=True, batchnorm=True, relu6=True, bn=bn)
        stages = torch7.graph_stages(ref["model"], dilate=opts.get("banks", {}).get("type") == "dilate",
                                     batchnorm=bn is not None)
        torch7.check_stages(stages, ref["mconf"], opts)
        return cls(stages, ref["is3D"], device=device, **opts), ref["mconf"]

    MODES = {"fp32": 0, "tf32": 1, "tf32x3": 2}

    def set_mode(self, mode):
        """'fp32' (CUDA-core FMA), 'tf32' or 'tf32x3' (wgmma tensor cores)."""
        self.ctx.check(self.ctx.lib.tfl_cnn_set_mode(self.ctx.h, self.h, self.MODES[mode]))

    def get_mode(self):
        m = self.ctx.lib.tfl_cnn_get_mode(self.h)
        return [k for k, v in self.MODES.items() if v == m][0]

    def __del__(self):
        try:
            if getattr(self, "h", None):
                self.ctx.lib.tfl_cnn_destroy(self.ctx.h, self.h)
                self.h = None
        except Exception:
            pass

    def forward(self, inputs, out=None, return_scale=False):
        """inputs = (pDiv, UDiv, flags) -> (p, U).  `out=(p, U)` writes in place (they may
        alias the inputs, which is what tfluids.simulate does, lib/simulate.lua:267-272)."""
        pDiv, UDiv, flags = inputs
        if out is None:
            p, U = torch.empty_like(pDiv), torch.empty_like(UDiv)
        else:
            p, U = out
        c = tfluids._ctx_for(pDiv)
        if c is not self.ctx:
            raise TflError("model and tensors live on different devices")
        sc = None
        scp = None
        if return_scale:
            sc = np.zeros(pDiv.size(0), np.float32)
            scp = sc.ctypes.data_as(C.POINTER(C.c_float))
        c.check(c.lib.tfl_cnn_project(c.h, self.h, tfluids._grid(pDiv), tfluids._grid(UDiv),
                                      tfluids._grid(flags), tfluids._grid(p), tfluids._grid(U),
                                      self.threshold, scp))
        self.last_scale = sc
        return p, U


def getModelInput(batch):
    """torch.getModelInput (lib/model.lua:421-423)."""
    return (batch["pDiv"], batch["UDiv"], batch["flags"])
