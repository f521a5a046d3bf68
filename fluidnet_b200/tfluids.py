"""Host-side mirror of the reference's `tfluids` Lua module (torch/tfluids/init.lua).

Same function names, argument order, defaults and assertion messages as the Lua wrappers;
tensors are torch CUDA float32 tensors (5-D, contiguous) whose storage is handed to
libtfl.so through the C ABI (include/tfl.h).  Temporaries live in the library's arena
(the Lua `getTempStorage`, init.lua:35-64), not in the caller.

There is no CPU path: a CPU tensor, a missing libtfl.so or a missing CUDA device raises.
"""
import ctypes as C

import torch

from . import _lib
from ._lib import Grid, TflError


class CellType:
    """tfluids.CellType (torch/tfluids/init.cu:108-124)."""
    TypeNone = 0
    TypeFluid = 1
    TypeObstacle = 2
    TypeEmpty = 4
    TypeInflow = 8
    TypeOutflow = 16
    TypeOpen = 32
    TypeStick = 128
    TypeReserved = 256
    TypeZeroPressure = 1 << 15


withCUDA = True
_contexts = {}


class Context:
    """One libtfl context per device; follows torch's current stream."""

    def __init__(self, device):
        self.lib = _lib.load()
        if not torch.cuda.is_available():
            raise TflError("fluidnet_b200 needs a CUDA device (no CPU fallback)")
        h = C.c_void_p()
        if self.lib.tfl_create(C.byref(h), int(device)) != 0:
            raise TflError("tfl_create failed on device %d" % device)
        self.h = h
        self.device = int(device)
        self._stream = None

    def use_current_stream(self):
        s = torch.cuda.current_stream(self.device).cuda_stream
        s = s if s != 0 else 1          # 0x1 == cudaStreamLegacy (torch's default stream)
        if s != self._stream:
            self.check(self.lib.tfl_set_stream(self.h, C.c_void_p(s)))
            self._stream = s

    def check(self, rc):
        if rc != 0:
            raise TflError(self.lib.tfl_last_error(self.h).decode())

    def launch_count(self):
        return int(self.lib.tfl_launch_count(self.h))

    def trace_faults(self, reset=True):
        v = C.c_int64(0)
        self.check(self.lib.tfl_trace_faults(self.h, C.byref(v), 1 if reset else 0))
        return v.value

    def set_slab(self, z_offset, global_nz, z_lo, z_hi):
        self.check(self.lib.tfl_set_slab(self.h, z_offset, global_nz, z_lo, z_hi))

    def clear_slab(self):
        self.check(self.lib.tfl_set_slab(self.h, 0, 0, 0, 0))


def context(device=None):
    if device is None:
        device = torch.cuda.current_device() if torch.cuda.is_available() else 0
    if isinstance(device, torch.device):
        device = device.index if device.index is not None else torch.cuda.current_device()
    if device not in _contexts:
        _contexts[device] = Context(device)
    return _contexts[device]


def _ctx_for(t):
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise TflError("tfluids: tensors must be CUDA tensors (there is no CPU path)")
    c = context(t.device.index)
    c.use_current_stream()
    return c


def _grid(t):
    assert t.dtype == torch.float32, "tfluids: tensors must be float32"
    return Grid(C.c_void_p(t.data_ptr()), t.size(0), t.size(1), t.size(2), t.size(3), t.size(4))


def _check_u_flags(U, flags):
    """The asserts shared by the Lua wrappers (e.g. init.lua:177-191)."""
    assert U.dim() == 5 and flags.dim() == 5, 'Dimension mismatch'
    assert flags.size(1) == 1, 'flags is not scalar'
    bsz, d, h, w = flags.size(0), flags.size(2), flags.size(3), flags.size(4)
    is3D = U.size(1) == 3
    if not is3D:
        assert d == 1, '2D velocity field but zdepth > 1'
        assert U.size(1) == 2, '2D velocity field must have only 2 channels'
    assert (U.size(0) == bsz and U.size(2) == d and U.size(3) == h and U.size(4) == w), 'Size mismatch'
    return is3D


def getDx(flags):
    """init.lua:560-565."""
    return 1.0 / max(flags.size(2), flags.size(3), flags.size(4))


def advectScalar(dt, s, U, flags, method=None, sDst=None, sampleOutsideFluid=None,
                 maccormackStrength=None, boundaryWidth=None):
    """init.lua:89-149."""
    method = method or "maccormackOurs"
    if sampleOutsideFluid is None:
        sampleOutsideFluid = False
    if maccormackStrength is None:
        maccormackStrength = 0.75
    assert s.dim() == 5 and U.dim() == 5 and flags.dim() == 5, 'Dimension mismatch'
    _check_u_flags(U, flags)
    assert s.size() == flags.size(), 'Size mismatch'
    assert s.is_contiguous() and U.is_contiguous() and flags.is_contiguous(), 'Input is not contiguous'
    if sDst is not None:
        assert sDst.dim() == 5, 'Size mismatch'
        assert sDst.is_contiguous(), 'Input is not contiguous'
        assert sDst.size() == s.size(), 'Size mismatch'
    c = _ctx_for(s)
    m = c.lib.tfl_advect_method_from_string(method.encode())
    if m < 0:
        raise TflError("advection method (%s) not supported (options are: euler, maccormack, rk2Ours, "
                       "rk3Ours, eulerOurs)" % method)
    gd = _grid(sDst) if sDst is not None else None
    c.check(c.lib.tfl_advect_scalar(c.h, float(dt), _grid(s), _grid(U), _grid(flags), m,
                                    1 if sampleOutsideFluid else 0, float(maccormackStrength),
                                    C.byref(gd) if gd is not None else None))


def advectVel(dt, U, flags, method=None, UDst=None, maccormackStrength=None, boundaryWidth=None):
    """init.lua:170-219."""
    method = method or "maccormackOurs"
    if maccormackStrength is None:
        maccormackStrength = 0.75
    _check_u_flags(U, flags)
    assert U.is_contiguous() and flags.is_contiguous(), 'Input is not contiguous'
    if UDst is not None:
        assert UDst.dim() == 5, 'Size mismatch'
        assert UDst.is_contiguous(), 'Input is not contiguous'
        assert UDst.size() == U.size(), 'Size mismatch'
    c = _ctx_for(U)
    m = c.lib.tfl_advect_method_from_string(method.encode())
    if m < 0:
        raise TflError("advection method (%s) not supported" % method)
    gd = _grid(UDst) if UDst is not None else None
    c.check(c.lib.tfl_advect_vel(c.h, float(dt), _grid(U), _grid(flags), m, float(maccormackStrength),
                                 C.byref(gd) if gd is not None else None))


def setWallBcsForward(U, flags):
    """init.lua:228-247."""
    _check_u_flags(U, flags)
    assert U.is_contiguous() and flags.is_contiguous()
    c = _ctx_for(U)
    c.check(c.lib.tfl_set_wall_bcs_forward(c.h, _grid(U), _grid(flags)))


def velocityDivergenceForward(U, flags, UDiv):
    """init.lua:256-279."""
    assert UDiv.dim() == 5, 'Dimension mismatch'
    _check_u_flags(U, flags)
    assert flags.size() == UDiv.size(), 'Size mismatch'
    assert U.is_contiguous() and flags.is_contiguous() and UDiv.is_contiguous(), 'Input is not contiguous'
    c = _ctx_for(U)
    c.check(c.lib.tfl_velocity_divergence_forward(c.h, _grid(U), _grid(flags), _grid(UDiv)))


def velocityUpdateForward(U, flags, p):
    """init.lua:324-349."""
    assert p.dim() == 5, 'Dimension mismatch'
    _check_u_flags(U, flags)
    assert p.size() == flags.size(), 'Size mismatch'
    assert U.is_contiguous() and flags.is_contiguous() and p.is_contiguous(), 'Input is not contiguous'
    c = _ctx_for(U)
    c.check(c.lib.tfl_velocity_update_forward(c.h, _grid(U), _grid(flags), _grid(p)))


def _gravity3(gravity):
    if isinstance(gravity, torch.Tensor):
        assert gravity.dim() == 1 and gravity.size(0) == 3, 'gravity must be a 3D vector (even in 2D).'
        vals = [float(v) for v in gravity.detach().cpu().float().tolist()]
    else:
        vals = [float(v) for v in gravity]
        assert len(vals) == 3, 'gravity must be a 3D vector (even in 2D).'
    return (C.c_float * 3)(*vals)


def addBuoyancy(U, flags, density, gravity, dt):
    """init.lua:442-471."""
    assert density.dim() == 5, 'Dimension mismatch'
    _check_u_flags(U, flags)
    assert density.size() == flags.size(), 'Size mismatch'
    assert U.is_contiguous() and flags.is_contiguous() and density.is_contiguous(), 'Input is not contiguous'
    assert isinstance(dt, (int, float)), 'time step must be a number'
    c = _ctx_for(U)
    c.check(c.lib.tfl_add_buoyancy(c.h, _grid(U), _grid(flags), _grid(density), _gravity3(gravity),
                                   float(dt)))


def addGravity(U, flags, gravity, dt):
    """init.lua:481-507."""
    _check_u_flags(U, flags)
    assert U.is_contiguous() and flags.is_contiguous(), 'Input is not contiguous'
    assert isinstance(dt, (int, float)), 'time step must be a number'
    c = _ctx_for(U)
    c.check(c.lib.tfl_add_gravity(c.h, _grid(U), _grid(flags), _gravity3(gravity), float(dt)))


def vorticityConfinement(U, flags, strength):
    """init.lua:394-431."""
    _check_u_flags(U, flags)
    assert U.is_contiguous() and flags.is_contiguous(), 'Input is not contiguous'
    assert isinstance(strength, (int, float))
    c = _ctx_for(U)
    c.check(c.lib.tfl_vorticity_confinement(c.h, _grid(U), _grid(flags), float(strength)))


def emptyDomain(flags, is3D, bnd=None):
    """init.lua:545-555."""
    bnd = bnd or 1
    assert flags.dim() == 5, 'Flags should be 5D'
    assert flags.size(1) == 1, 'Flags should be a scalar'
    assert ((not is3D or flags.size(2) >= bnd * 2 + 1) and flags.size(3) >= bnd * 2 + 1 and
            flags.size(4) >= bnd * 2 + 1), 'simulation domain not big enough!'
    c = _ctx_for(flags)
    c.check(c.lib.tfl_empty_domain(c.h, _grid(flags), 1 if is3D else 0, int(bnd)))
    return flags


def flagsToOccupancy(flags, occupancy):
    """init.lua:571-576; raises like the CPU reference on unsupported cells
    (generic/tfluids.cc:194-207)."""
    assert flags.dim() == 5 and occupancy.dim() == 5
    assert flags.size(1) == 1 and flags.size() == occupancy.size()
    c = _ctx_for(flags)
    bad = C.c_int64(0)
    c.check(c.lib.tfl_flags_to_occupancy(c.h, _grid(flags), _grid(occupancy), C.byref(bad)))
    if bad.value:
        raise TflError("ERROR: unsupported flag cell found!")


def solveLinearSystemJacobi(p, flags, div, is3D, pTol=None, maxIter=None, verbose=None):
    """init.lua:693-734. Returns the max residual across the batch."""
    assert p.dim() == 5 and flags.dim() == 5 and div.dim() == 5, 'Dimension mismatch'
    assert flags.size(1) == 1, 'flags is not scalar'
    assert p.size() == flags.size(), 'size mismatch'
    assert div.size() == flags.size(), 'size mismatch'
    if not is3D:
        assert flags.size(2) == 1, 'd > 1 for a 2D domain'
    pTol = 1e-5 if pTol is None else pTol
    maxIter = 1000 if maxIter is None else maxIter
    assert p.is_contiguous() and flags.is_contiguous() and div.is_contiguous()
    c = _ctx_for(p)
    res = C.c_float(0)
    it = C.c_int(0)
    c.check(c.lib.tfl_solve_linear_system_jacobi(c.h, _grid(p), _grid(flags), _grid(div),
                                                 1 if is3D else 0, float(pTol), int(maxIter),
                                                 C.byref(res), C.byref(it)))
    solveLinearSystemJacobi.last_iterations = it.value
    return float(res.value)


def solveLinearSystemJacobiDevice(p, flags, div, is3D, pTol, maxIter):
    """solveLinearSystemJacobi with its results left on the device: returns (residual [1] float32, iterations [1]
    int32) CUDA tensors, written in stream order on torch's current stream.  Does not wait for the device on
    L2-resident 3-D grids or inside a CUDA graph capture (capture it once the same solve has run outside the
    capture); other grids outside a capture wait once per chunk of up to 256 sweeps (tfl.h)."""
    assert p.dim() == 5 and flags.dim() == 5 and div.dim() == 5, 'Dimension mismatch'
    assert flags.size(1) == 1, 'flags is not scalar'
    assert p.size() == flags.size(), 'size mismatch'
    assert div.size() == flags.size(), 'size mismatch'
    if not is3D:
        assert flags.size(2) == 1, 'd > 1 for a 2D domain'
    assert p.is_contiguous() and flags.is_contiguous() and div.is_contiguous()
    c = _ctx_for(p)
    residual = torch.empty(1, dtype=torch.float32, device=p.device)
    iterations = torch.empty(1, dtype=torch.int32, device=p.device)
    c.check(c.lib.tfl_solve_linear_system_jacobi_dev(c.h, _grid(p), _grid(flags), _grid(div), 1 if is3D else 0,
                                                     float(pTol), int(maxIter), C.c_void_p(residual.data_ptr()),
                                                     C.c_void_p(iterations.data_ptr())))
    return residual, iterations


def solveLinearSystemPCG(p, flags, div, is3D, tol=None, maxIter=None, precondType=None, verbose=None):
    """init.lua:645-676 (same argument order and defaults). Returns the max residual across the
    batch elements and connected fluid components."""
    assert p.dim() == 5 and flags.dim() == 5 and div.dim() == 5, 'Dimension mismatch'
    assert flags.size(1) == 1, 'flags is not scalar'
    assert p.size() == flags.size(), 'size mismatch'
    assert div.size() == flags.size(), 'size mismatch'
    if not is3D:
        assert flags.size(2) == 1, 'd > 1 for a 2D domain'
    precondType = precondType or 'ic0'
    tol = 1e-6 if tol is None else tol
    maxIter = 1000 if maxIter is None else maxIter
    assert p.is_contiguous() and flags.is_contiguous() and div.is_contiguous()
    c = _ctx_for(p)
    kind = c.lib.tfl_precond_from_string(precondType.encode())
    if kind < 0:
        raise TflError("Incorrect preconType ('none', 'ic0', 'ilu0')")
    res = C.c_float(0)
    it = C.c_int(0)
    c.check(c.lib.tfl_solve_linear_system_pcg(c.h, _grid(p), _grid(flags), _grid(div), 1 if is3D else 0, kind,
                                              float(tol), int(maxIter), C.byref(res), C.byref(it)))
    solveLinearSystemPCG.last_iterations = it.value
    return float(res.value)


def normalizePressureMean(p, flags, is3D):
    """init.lua:747-765: remove the mean of p over every connected fluid component (on the device;
    the reference round-trips through the host)."""
    assert p.dim() == 5 and flags.dim() == 5 and p.size() == flags.size()
    assert p.is_contiguous() and flags.is_contiguous()
    c = _ctx_for(p)
    c.check(c.lib.tfl_normalize_pressure_mean(c.h, _grid(p), _grid(flags), 1 if is3D else 0))


def volumetricUpSamplingNearestForward(ratio, input, output):
    """init.lua:618-622."""
    assert input.dim() == 5 and output.dim() == 5, 'ERROR: input and output must be dim 5'
    assert input.is_contiguous() and output.is_contiguous()
    c = _ctx_for(input)
    c.check(c.lib.tfl_volumetric_up_sampling_nearest_forward(c.h, int(ratio), _grid(input), _grid(output)))


def rectangularBlur(src, blurRad, is3D, dst):
    """init.lua:583-596."""
    assert src.dim() == 5 and dst.dim() == 5
    assert src.size() == dst.size()
    assert blurRad > 0 and int(blurRad) == blurRad, 'blurRad must be a positive, non-zero integer'
    assert src.is_contiguous() and dst.is_contiguous()
    c = _ctx_for(src)
    c.check(c.lib.tfl_rectangular_blur(c.h, _grid(src), int(blurRad), 1 if is3D else 0, _grid(dst)))


def signedDistanceField(flags, searchRad, is3D, dst):
    """init.lua:604-614."""
    assert flags.dim() == 5 and dst.dim() == 5
    assert flags.size() == dst.size()
    assert flags.is_contiguous() and dst.is_contiguous()
    assert flags.size(1) == 1, 'flags must be scalar'
    assert searchRad > 0 and int(searchRad) == searchRad, 'searchRad must be a positive, non-zero integer'
    c = _ctx_for(flags)
    c.check(c.lib.tfl_signed_distance_field(c.h, _grid(flags), int(searchRad), 1 if is3D else 0, _grid(dst)))


def velocityDivergenceBackward(U, flags, gradOutput, gradU):
    """init.lua:288-314."""
    assert U.dim() == 5 and flags.dim() == 5 and gradOutput.dim() == 5 and gradU.dim() == 5, 'Dimension mismatch'
    assert flags.size(1) == 1, 'flags is not scalar'
    assert gradU.size() == U.size() and gradOutput.size() == flags.size(), 'Size mismatch'
    assert all(t.is_contiguous() for t in (U, flags, gradOutput, gradU)), 'Input is not contiguous'
    c = _ctx_for(U)
    c.check(c.lib.tfl_velocity_divergence_backward(c.h, _grid(U), _grid(flags), _grid(gradOutput), _grid(gradU)))


def velocityUpdateBackward(U, flags, p, gradOutput, gradP):
    """init.lua:358-384."""
    assert all(t.dim() == 5 for t in (U, flags, p, gradOutput, gradP)), 'Dimension mismatch'
    assert flags.size(1) == 1, 'flags is not scalar'
    assert gradP.size() == p.size() and gradOutput.size() == U.size(), 'Size mismatch'
    assert all(t.is_contiguous() for t in (U, flags, p, gradOutput, gradP)), 'Input is not contiguous'
    c = _ctx_for(U)
    c.check(c.lib.tfl_velocity_update_backward(c.h, _grid(U), _grid(flags), _grid(p), _grid(gradOutput), _grid(gradP)))


def volumetricUpSamplingNearestBackward(ratio, input, gradOutput, gradInput):
    """init.lua:623-627."""
    assert input.dim() == 5 and gradOutput.dim() == 5 and gradInput.dim() == 5
    c = _ctx_for(input)
    c.check(c.lib.tfl_volumetric_up_sampling_nearest_backward(c.h, int(ratio), _grid(input), _grid(gradOutput),
                                                              _grid(gradInput)))


def applyBC(x, invMask, bc):
    """x:cmul(invMask); x:add(bc) -- the cutorch pair in setConstVals (lib/simulate.lua:136-158)."""
    c = _ctx_for(x)
    c.check(c.lib.tfl_apply_bc(c.h, _grid(x), _grid(invMask), _grid(bc)))


def clamp(x, lo, hi):
    """U:clamp(lo, hi) (lib/simulate.lua:326)."""
    c = _ctx_for(x)
    c.check(c.lib.tfl_clamp(c.h, _grid(x), float(lo), float(hi)))
