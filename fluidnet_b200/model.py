"""Pressure-projection model (forward only) -- mirror of torch/lib/model.lua.

`ProjectionModel` plays the role of the nngraph module built by torch.defineModelGraph
(lib/model.lua:27-401) for the 'default' input set {pDiv, div, flags}: `forward({pDiv, UDiv,
flags})` returns `{p, U}` (lib/model.lua:421-450).  The whole graph runs inside libtfl.so
(tfl_cnn_project); weights are plain float32 arrays in Torch layout [cout][cin][kz][ky][kx].
"""
import ctypes as C

import numpy as np
import torch

from . import tfluids
from ._lib import TflError


def default_layers(is3D):
    """(cin, cout, k) of the 'default' modelType (lib/model.lua:179-186 2-D, :219-226 3-D)."""
    if is3D:
        return [(3, 8, 3), (8, 8, 3), (8, 8, 3), (8, 8, 1), (8, 1, 1)]
    return [(3, 16, 3), (16, 16, 3), (16, 16, 3), (16, 16, 3), (16, 1, 1)]


class ProjectionModel:
    def __init__(self, layers, is3D, device=None, normalizeInputThreshold=1e-5, pool=None, up=None,
                 poolType="avg", nonlinType="relu"):
        """layers: [(weight ndarray [cout * up^d][cin][kz][ky][kx], bias ndarray [cout * up^d]), ...]
        pool / up: per-layer pooling and ConvolutionUpsample sizes of the 'tog' graph (lib/model.lua:164-226),
        None = all 1 ('default', 'yang'); poolType 'avg' | 'max'; nonlinType 'relu' | 'sigmoid'."""
        self.is3D = bool(is3D)
        self.threshold = float(normalizeInputThreshold)
        self.ctx = tfluids.context(device)
        n = len(layers)
        pool = [1] * n if pool is None else [int(v) for v in pool]
        up = [1] * n if up is None else [int(v) for v in up]
        assert len(pool) == n and len(up) == n
        assert poolType in ("avg", "max") and nonlinType in ("relu", "sigmoid")
        self._keep = []
        cin = (C.c_int32 * n)()
        cout = (C.c_int32 * n)()
        ks = (C.c_int32 * n)()
        cpool = (C.c_int32 * n)(*pool)
        cup = (C.c_int32 * n)(*up)
        wp = (C.POINTER(C.c_float) * n)()
        bp = (C.POINTER(C.c_float) * n)()
        for l, (w, b) in enumerate(layers):
            w = np.ascontiguousarray(w, dtype=np.float32)
            b = np.ascontiguousarray(b, dtype=np.float32)
            assert w.ndim == 5 and b.ndim == 1 and b.shape[0] == w.shape[0]
            assert w.shape[3] == w.shape[4] and w.shape[2] == (w.shape[4] if is3D else 1)
            fan = up[l] ** (3 if is3D else 2)
            assert w.shape[0] % fan == 0, "ConvolutionUpsample layer: cout must be a multiple of up^d"
            self._keep += [w, b]
            cout[l], cin[l], ks[l] = w.shape[0] // fan, w.shape[1], w.shape[4]
            wp[l] = w.ctypes.data_as(C.POINTER(C.c_float))
            bp[l] = b.ctypes.data_as(C.POINTER(C.c_float))
        h = C.c_void_p()
        self.ctx.check(self.ctx.lib.tfl_cnn_create_graph(self.ctx.h, 1 if is3D else 0, n, cin, cout, ks, cpool, cup,
                                                         1 if poolType == "max" else 0,
                                                         1 if nonlinType == "sigmoid" else 0, wp, bp, C.byref(h)))
        self.h = h
        self.last_scale = None

    @classmethod
    def from_reference_file(cls, model_path, mconf_path=None, device=None):
        """A model saved by the reference (torch/lib/save_model.lua: Torch7 binary network + `_mconf.bin`),
        read without Torch7 (fluidnet_b200/torch7.py).  Returns (model, mconf)."""
        from . import torch7
        ref = torch7.load_reference_model(model_path, mconf_path)
        thr = ref["mconf"].get("normalizeInputThreshold", 1e-5)
        return cls(ref["layers"], ref["is3D"], device=device, normalizeInputThreshold=thr), ref["mconf"]

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
