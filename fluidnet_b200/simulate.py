"""Mirror of torch/lib/simulate.lua: `simulate(conf, mconf, batch, model, outputDiv)` advances
the fluid state in `batch` by one time step with the same operator sequence
(lib/simulate.lua:175-327), and `createPlumeBCs` / `removeBCs` build the boundary-condition
tensors (lib/simulate.lua:33-123).

`batch` is a dict of torch CUDA tensors with the reference's keys: pDiv, UDiv, flags,
density (+ UBC, UBCInvMask, densityBC, densityBCInvMask, pBC, pBCInvMask).  mconf is a
dict with the reference's keys (dt, advectionMethod, maccormackStrength, buoyancyScale,
gravityScale, gravity, vorticityConfinementAmp, simMethod, maxIter, is3D).

Two execution modes produce identical results:
  * operator by operator through `tfluids.*` (default for simMethod ~= 'convnet'), and
  * `simulate_fused`: one C-ABI call (tfl_simulate_step) that enqueues the whole step.
"""
import ctypes as C
import math

import torch

from . import tfluids
from ._lib import Grid, MConf, State


def getPUFlagsDensityReference(batch):
    """lib/simulate.lua:25-31."""
    density = batch.get("density", batch.get("densityDiv"))
    return batch["pDiv"], batch["UDiv"], batch["flags"], density


def removeBCs(batch):
    for k in ("pBC", "pBCInvMask", "UBC", "UBCInvMask", "densityBC", "densityBCInvMask"):
        batch.pop(k, None)


def createPlumeBCs(batch, densityVal, uScale, rad):
    """lib/simulate.lua:47-123 (built on the host, uploaded once)."""
    U = batch["UDiv"]
    assert batch.get("density") is not None, 'plume BCs require a density field to be specified'
    assert isinstance(densityVal, (list, tuple)) and len(densityVal) == 1, \
        'there should be a single density value'
    assert U.dim() == 5
    assert U.size(0) == 1, 'Only single batch allowed.'
    xdim, ydim, zdim = U.size(4), U.size(3), U.size(2)
    is3D = U.size(1) == 3
    if not is3D:
        assert zdim == 1
    UBC = torch.zeros(U.shape, dtype=torch.float32)
    UInv = torch.ones(U.shape, dtype=torch.float32)
    dBC = torch.zeros(batch["density"].shape, dtype=torch.float32)
    dInv = torch.ones(batch["density"].shape, dtype=torch.float32)
    centerX = xdim // 2
    centerZ = max(zdim // 2, 1)
    plumeRad = math.floor(xdim * rad)
    x = torch.arange(1, xdim + 1).view(1, xdim)
    z = torch.arange(1, zdim + 1).view(zdim, 1)
    inside = ((centerX - x) ** 2 + (centerZ - z) ** 2) <= plumeRad * plumeRad     # [z][x]
    for y in range(4):                       # Lua y = 1..4
        UInv[0, :, :, y, :] = 0
        UBC[0, 1, :, y, :] = torch.where(inside, torch.tensor(float(uScale)), torch.tensor(0.0))
        dBC[0, 0, :, y, :] = torch.where(inside, torch.tensor(float(densityVal[0])), torch.tensor(0.0))
        dInv[0, 0, :, y, :] = torch.where(inside, torch.tensor(0.0), torch.tensor(1.0))
    dev = U.device
    batch["pBC"] = None
    batch["pBCInvMask"] = None
    batch["UBC"], batch["UBCInvMask"] = UBC.to(dev), UInv.to(dev)
    batch["densityBC"], batch["densityBCInvMask"] = dBC.to(dev), dInv.to(dev)


def setConstVals(batch, p, U, flags, density):
    """lib/simulate.lua:130-160."""
    if batch.get("pBC") is not None or batch.get("pBCInvMask") is not None:
        tfluids.applyBC(p, batch["pBCInvMask"], batch["pBC"])
    if batch.get("UBC") is not None or batch.get("UBCInvMask") is not None:
        tfluids.applyBC(U, batch["UBCInvMask"], batch["UBC"])
    if batch.get("densityBC") is not None or batch.get("densityBCInvMask") is not None:
        tfluids.applyBC(density, batch["densityBCInvMask"], batch["densityBC"])


def _gravity(mconf):
    g = mconf.get("gravity")
    if g is None:
        return [0.0, 1.0, 0.0]                                # lib/simulate.lua:204-213
    if isinstance(g, torch.Tensor):
        return [float(v) for v in g.cpu().tolist()]
    return [float(v) for v in g]


def _f32(x):
    return torch.tensor(x, dtype=torch.float32).item()


def simulate(conf, mconf, batch, model=None, outputDiv=False):
    """tfluids.simulate (lib/simulate.lua:175-327), operator by operator."""
    p, U, flags, density = getPUFlagsDensityReference(batch)
    if density is not None:
        tfluids.advectScalar(mconf["dt"], density, U, flags, mconf.get("advectionMethod"), None, False,
                             mconf.get("maccormackStrength"))
    tfluids.advectVel(mconf["dt"], U, flags, mconf.get("advectionMethod"), None,
                      mconf.get("maccormackStrength"))
    setConstVals(batch, p, U, flags, density)
    dx = tfluids.getDx(flags)
    if density is not None and mconf.get("buoyancyScale", 0) > 0:
        k = _f32(-(dx / 4) * mconf["buoyancyScale"])           # gravity:mul(scalar), float tensor op
        g = [_f32(_f32(v) * k) for v in _gravity(mconf)]
        tfluids.addBuoyancy(U, flags, density, g, mconf["dt"])
    if mconf.get("gravityScale", 0) > 0:
        k = _f32((-dx / 4) * mconf["gravityScale"])
        g = [_f32(_f32(v) * k) for v in _gravity(mconf)]
        tfluids.addGravity(U, flags, g, mconf["dt"])
    if mconf.get("vorticityConfinementAmp", 0) > 0:
        tfluids.vorticityConfinement(U, flags, dx * mconf["vorticityConfinementAmp"])
    if outputDiv:
        return
    simMethod = mconf.get("simMethod") or "convnet"
    if simMethod != "convnet":
        tfluids.setWallBcsForward(U, flags)
    setConstVals(batch, p, U, flags, density)
    if simMethod == "convnet":
        model.forward((p, U, flags), out=(p, U))               # p:copy(pPred); U:copy(UPred)
    else:
        if batch.get("div") is None:
            batch["div"] = torch.empty_like(p)
        tfluids.velocityDivergenceForward(U, flags, batch["div"])
        if simMethod == "jacobi":
            tfluids.solveLinearSystemJacobi(p, flags, batch["div"], mconf["is3D"], 0,
                                            mconf.get("maxIter") or 100)
        elif simMethod == "pcg":
            tfluids.solveLinearSystemPCG(p, flags, batch["div"], mconf["is3D"], 1e-4,
                                         mconf.get("maxIter") or 100, "ic0")
        else:
            raise ValueError("mconf.simMethod (%s) is not a valid option" % simMethod)
        tfluids.velocityUpdateForward(U, flags, p)
    setConstVals(batch, p, U, flags, density)
    tfluids.clamp(U, -1e6, 1e6)


_SIM = {"convnet": 0, "jacobi": 1, "pcg": 2}


def make_mconf(mconf):
    m = MConf()
    m.dt = float(mconf["dt"])
    m.advection_method = tfluids.context().lib.tfl_advect_method_from_string(
        (mconf.get("advectionMethod") or "maccormackOurs").encode())
    ms = mconf.get("maccormackStrength")
    m.maccormack_strength = 0.75 if ms is None else float(ms)
    m.buoyancy_scale = float(mconf.get("buoyancyScale", 0) or 0)
    m.gravity_scale = float(mconf.get("gravityScale", 0) or 0)
    g = _gravity(mconf)
    m.gravity[0], m.gravity[1], m.gravity[2] = g
    m.vorticity_confinement_amp = float(mconf.get("vorticityConfinementAmp", 0) or 0)
    m.sim_method = _SIM[mconf.get("simMethod") or "convnet"]
    m.max_iter = int(mconf.get("maxIter") or 0)
    m.normalize_input_threshold = float(mconf.get("normalizeInputThreshold", 1e-5))
    return m


def make_state(batch):
    s = State()
    zero = Grid(None, 0, 0, 0, 0, 0)
    for name, key in (("p", "pDiv"), ("U", "UDiv"), ("flags", "flags"), ("density", "density"),
                      ("U_bc", "UBC"), ("U_bc_inv_mask", "UBCInvMask"), ("density_bc", "densityBC"),
                      ("density_bc_inv_mask", "densityBCInvMask"), ("p_bc", "pBC"),
                      ("p_bc_inv_mask", "pBCInvMask"), ("div", "div")):
        t = batch.get(key)
        setattr(s, name, tfluids._grid(t) if t is not None else zero)
    return s


def simulate_fused(conf, mconf, batch, model=None):
    """Same step as `simulate`, enqueued by one C-ABI call (tfl_simulate_step)."""
    p = batch["pDiv"]
    if (mconf.get("simMethod") or "convnet") != "convnet" and batch.get("div") is None:
        batch["div"] = torch.empty_like(p)
    c = tfluids._ctx_for(p)
    st = make_state(batch)
    mc = make_mconf(mconf)
    if model is not None:
        # one source for the input-scale threshold: the model's (what `simulate` uses through model.forward)
        mc.normalize_input_threshold = float(model.threshold)
    c.check(c.lib.tfl_simulate_step(c.h, C.byref(st), C.byref(mc), model.h if model is not None else None))


class StepGraph:
    """One simulate_fused call captured as a CUDA graph (tfl_step_graph_*): `launch()` replays it on the
    batch tensors it was captured with.  Needs a non-default current stream and one earlier step."""

    def __init__(self, mconf, batch, model=None):
        p = batch["pDiv"]
        if (mconf.get("simMethod") or "convnet") != "convnet" and batch.get("div") is None:
            batch["div"] = torch.empty_like(p)
        self.ctx = tfluids._ctx_for(p)
        self.batch, self.model = batch, model          # keep the captured tensors alive
        st = make_state(batch)
        mc = make_mconf(mconf)
        if model is not None:
            mc.normalize_input_threshold = float(model.threshold)
        h = C.c_void_p()
        self.ctx.check(self.ctx.lib.tfl_step_graph_create(self.ctx.h, C.byref(st), C.byref(mc),
                                                          model.h if model is not None else None, C.byref(h)))
        self.h = h

    def launch(self):
        self.ctx.use_current_stream()
        self.ctx.check(self.ctx.lib.tfl_step_graph_launch(self.ctx.h, self.h))

    def pcg_status(self):
        """(residual, iterations) of the last replay's PCG solve, as solveLinearSystemPCG returns them (-inf, 0
        without a component to solve); iterations is -1 for a step without a PCG solve.  Synchronises.  Raises
        TflError with the direct solve's message for the first replay since the previous call whose solve failed."""
        self.ctx.use_current_stream()
        res, it = C.c_float(0.0), C.c_int32(0)
        self.ctx.check(self.ctx.lib.tfl_step_graph_pcg_status(self.ctx.h, self.h, C.byref(res), C.byref(it)))
        return res.value, it.value

    def close(self):
        if self.h:
            self.ctx.lib.tfl_step_graph_destroy(self.ctx.h, self.h)
            self.h = None
