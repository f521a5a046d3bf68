"""TEST INFRASTRUCTURE ONLY (see oracle/__init__.py)."""
import ctypes as C
import math
import os
import subprocess

import numpy as np

from .model import model_forward

HERE = os.path.dirname(os.path.abspath(__file__))
ORACLE_SO = os.path.join(HERE, "liboracle.so")
REF_SO = os.path.join(HERE, "_ref", "libtfluids_ref.so")
REF_SRC = "/root/reference/torch/tfluids"


class CellType:
    """tfluids/third_party/cell_type.h:22-33."""
    TypeNone = 0
    TypeFluid = 1
    TypeObstacle = 2
    TypeEmpty = 4
    TypeInflow = 8
    TypeOutflow = 16
    TypeOpen = 32
    TypeStick = 128


# tfluids/generic/advect_type.cc:19-38
ADVECT_METHODS = {"euler": 0, "maccormack": 1, "eulerOurs": 2, "rk2Ours": 3, "rk3Ours": 4,
                  "maccormackOurs": 5}


def build(force=False):
    """Compile the checkers (building the checker is not using it)."""
    need_oracle = force or not os.path.exists(ORACLE_SO) or (
        os.path.getmtime(ORACLE_SO) < os.path.getmtime(os.path.join(HERE, "tfluids_oracle.c")))
    if need_oracle:
        subprocess.check_call(["make", "-s", "-C", HERE, "oracle"])
    if os.path.isdir(REF_SRC):
        drv = os.path.join(HERE, "ref_shim", "ref_driver.cc")
        if force or not os.path.exists(REF_SO) or os.path.getmtime(REF_SO) < os.path.getmtime(drv):
            subprocess.check_call(["make", "-s", "-C", HERE, "ref"])


def have_reference():
    return os.path.exists(REF_SO)


def _f32(a):
    a = np.ascontiguousarray(a, dtype=np.float32)
    return a


def _ptr(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


class _Dims(C.Structure):
    _fields_ = [("nb", C.c_int), ("nz", C.c_int), ("ny", C.c_int), ("nx", C.c_int),
                ("is3d", C.c_int)]


def _dims(flags, is3d):
    b, c, z, y, x = flags.shape
    assert c == 1
    return _Dims(b, z, y, x, 1 if is3d else 0)


def _is3d(U):
    assert U.ndim == 5 and U.shape[1] in (2, 3)
    return U.shape[1] == 3


class Oracle:
    """Our C restatement (oracle/tfluids_oracle.c)."""
    name = "oracle"

    def __init__(self):
        build()
        self.lib = C.CDLL(ORACLE_SO)
        L = self.lib
        L.orc_jacobi.restype = C.c_float
        L.orc_sample_std.restype = C.c_float
        L.orc_get_dx.restype = C.c_float
        L.orc_trace_faults.restype = C.c_long
        L.orc_flags_to_occupancy.restype = C.c_long

    def num_threads(self):
        return int(self.lib.orc_num_threads())

    def trace_faults(self):
        return int(self.lib.orc_trace_faults())

    # -- operators (names follow torch/tfluids/init.lua) ---------------------------------
    def emptyDomain(self, flags, is3D, bnd=1):
        assert flags.dtype == np.float32 and flags.flags.c_contiguous
        d = _dims(flags, is3D)
        self.lib.orc_empty_domain(_ptr(flags), C.byref(d), C.c_int(bnd))
        return flags

    def flagsToOccupancy(self, flags):
        flags = _f32(flags)
        occ = np.empty_like(flags)
        bad = self.lib.orc_flags_to_occupancy(_ptr(flags), _ptr(occ), C.c_long(flags.size))
        if bad:
            raise RuntimeError("ERROR: unsupported flag cell found!")
        return occ

    def advectScalar(self, dt, s, U, flags, method="maccormackOurs", sampleOutsideFluid=False,
                     maccormackStrength=0.75):
        s, U, flags = _f32(s), _f32(U), _f32(flags)
        is3d = _is3d(U)
        d = _dims(flags, is3d)
        dst = np.full_like(s, np.float32(123.0))
        fwd = np.full_like(s, np.float32(123.0))
        bwd = np.full_like(s, np.float32(123.0))
        fpos = np.zeros_like(U)
        bpos = np.zeros_like(U)
        self.lib.orc_advect_scalar(C.c_float(dt), _ptr(s), _ptr(U), _ptr(flags), C.byref(d),
                                   C.c_int(ADVECT_METHODS[method]),
                                   C.c_int(1 if sampleOutsideFluid else 0),
                                   C.c_float(maccormackStrength), _ptr(dst), _ptr(fwd), _ptr(bwd),
                                   _ptr(fpos), _ptr(bpos))
        return dst

    def advectVel(self, dt, U, flags, method="maccormackOurs", maccormackStrength=0.75):
        U, flags = _f32(U), _f32(flags)
        d = _dims(flags, _is3d(U))
        dst = np.full_like(U, np.float32(123.0))
        fwd = np.full_like(U, np.float32(123.0))
        bwd = np.full_like(U, np.float32(123.0))
        self.lib.orc_advect_vel(C.c_float(dt), _ptr(U), _ptr(flags), C.byref(d),
                                C.c_int(ADVECT_METHODS[method]), C.c_float(maccormackStrength),
                                _ptr(dst), _ptr(fwd), _ptr(bwd))
        return dst

    def setWallBcsForward(self, U, flags, as_mask_multiply=False):
        assert U.dtype == np.float32 and U.flags.c_contiguous
        flags = _f32(flags)
        d = _dims(flags, _is3d(U))
        self.lib.orc_set_wall_bcs(_ptr(U), _ptr(flags), C.byref(d),
                                  C.c_int(1 if as_mask_multiply else 0))

    def velocityDivergenceForward(self, U, flags):
        U, flags = _f32(U), _f32(flags)
        d = _dims(flags, _is3d(U))
        div = np.full_like(flags, np.float32(123.0))
        self.lib.orc_velocity_divergence(_ptr(U), _ptr(flags), _ptr(div), C.byref(d))
        return div

    def velocityUpdateForward(self, U, flags, p):
        assert U.dtype == np.float32 and U.flags.c_contiguous
        flags, p = _f32(flags), _f32(p)
        d = _dims(flags, _is3d(U))
        self.lib.orc_velocity_update(_ptr(U), _ptr(flags), _ptr(p), C.byref(d))

    def addBuoyancy(self, U, flags, density, gravity, dt):
        assert U.dtype == np.float32 and U.flags.c_contiguous
        flags, density = _f32(flags), _f32(density)
        g = _f32(np.asarray(gravity, dtype=np.float32).reshape(3))
        d = _dims(flags, _is3d(U))
        self.lib.orc_add_buoyancy(_ptr(U), _ptr(flags), _ptr(density), _ptr(g), C.c_float(dt),
                                  C.byref(d))

    def addGravity(self, U, flags, gravity, dt):
        assert U.dtype == np.float32 and U.flags.c_contiguous
        flags = _f32(flags)
        g = _f32(np.asarray(gravity, dtype=np.float32).reshape(3))
        d = _dims(flags, _is3d(U))
        self.lib.orc_add_gravity(_ptr(U), _ptr(flags), _ptr(g), C.c_float(dt), C.byref(d))

    def vorticityConfinement(self, U, flags, strength):
        assert U.dtype == np.float32 and U.flags.c_contiguous
        flags = _f32(flags)
        d = _dims(flags, _is3d(U))
        b, c, z, y, x = U.shape
        centered = np.zeros_like(U)
        curl = np.zeros((b, 3, z, y, x), np.float32)
        cnorm = np.zeros((b, 1, z, y, x), np.float32)
        force = np.zeros_like(U)
        self.lib.orc_vorticity_confinement(_ptr(U), _ptr(flags), C.c_float(strength), C.byref(d),
                                           _ptr(centered), _ptr(curl), _ptr(cnorm), _ptr(force))

    def solveLinearSystemJacobi(self, p, flags, div, is3D, pTol=1e-5, maxIter=1000):
        assert p.dtype == np.float32 and p.flags.c_contiguous
        flags, div = _f32(flags), _f32(div)
        d = _dims(flags, is3D)
        prev = np.empty_like(p)
        it = C.c_int(0)
        res = self.lib.orc_jacobi(_ptr(p), _ptr(flags), _ptr(div), C.byref(d), C.c_float(pTol),
                                  C.c_int(maxIter), _ptr(prev), C.byref(it))
        self.last_jacobi_iters = it.value
        return float(res)

    PRECOND = {"none": 0, "ilu0": 1, "ic0": 2}

    def solveLinearSystemPCG(self, p, flags, div, is3D, tol=1e-6, maxIter=1000, precondType="ic0"):
        """tfluids.solveLinearSystemPCG (tfluids/init.lua:645-676); returns the max residual."""
        assert p.dtype == np.float32 and p.flags.c_contiguous
        flags, div = _f32(flags), _f32(div)
        d = _dims(flags, is3D)
        res, it = C.c_float(0), C.c_int(0)
        rc = self.lib.orc_pcg(_ptr(p), _ptr(flags), _ptr(div), C.byref(d), C.c_int(self.PRECOND[precondType]),
                              C.c_float(tol), C.c_int(maxIter), C.byref(res), C.byref(it))
        if rc:
            raise RuntimeError("Non fluid cell found in a connected component")
        self.last_pcg_iters = it.value
        return float(res.value)

    def findConnectedFluidComponents(self, flags, is3D, ibatch=0):
        """(components [z][y][x] int32, sizes) of one batch element."""
        flags = _f32(flags)
        d = _dims(flags, is3D)
        comp = np.empty(flags.shape[2:], np.int32)
        sizes = np.zeros(comp.size + 1, np.int32)
        n = self.lib.orc_find_components(_ptr(flags), C.byref(d), C.c_int(ibatch), _ptr(comp), _ptr(sizes),
                                         C.c_int(sizes.size))
        return comp, sizes[:n].copy()

    # -- operators of tfluids/init.lua around the step ("next" rows) ----------------------------
    def velocityDivergenceBackward(self, U, flags, gradOutput):
        flags, go = _f32(flags), _f32(gradOutput)
        d = _dims(flags, _is3d(U))
        gU = np.empty_like(_f32(U))
        self.lib.orc_velocity_divergence_backward(_ptr(flags), _ptr(go), _ptr(gU), C.byref(d))
        return gU

    def velocityUpdateBackward(self, U, flags, p, gradOutput):
        flags, go = _f32(flags), _f32(gradOutput)
        d = _dims(flags, _is3d(U))
        gp = np.empty_like(flags)
        self.lib.orc_velocity_update_backward(_ptr(flags), _ptr(go), _ptr(gp), C.byref(d))
        return gp

    def volumetricUpSamplingNearestBackward(self, ratio, x, gradOutput):
        go = _f32(gradOutput)
        nb, nf, nz, ny, nx = x.shape
        gi = np.empty(x.shape, np.float32)
        self.lib.orc_upsample_nearest_backward(_ptr(go), _ptr(gi), C.c_int(nb), C.c_int(nf), C.c_int(nz), C.c_int(ny),
                                               C.c_int(nx), C.c_int(ratio))
        return gi

    def volumetricUpSamplingNearestForward(self, ratio, x):
        x = _f32(x)
        nb, nf, nz, ny, nx = x.shape
        out = np.empty((nb, nf, nz * ratio, ny * ratio, nx * ratio), np.float32)
        self.lib.orc_upsample_nearest(_ptr(x), _ptr(out), C.c_int(nb), C.c_int(nf), C.c_int(nz), C.c_int(ny),
                                      C.c_int(nx), C.c_int(ratio))
        return out

    def rectangularBlur(self, src, blurRad, is3D):
        src = _f32(src)
        dst, tmp = np.empty_like(src), np.empty_like(src)
        nb, nf, nz, ny, nx = src.shape
        self.lib.orc_rectangular_blur(_ptr(src), C.c_int(blurRad), C.c_int(1 if is3D else 0), _ptr(dst), _ptr(tmp),
                                      C.c_int(nb), C.c_int(nf), C.c_int(nz), C.c_int(ny), C.c_int(nx))
        return dst

    def signedDistanceField(self, flags, searchRad, is3D):
        flags = _f32(flags)
        d = _dims(flags, is3D)
        dst = np.empty_like(flags)
        self.lib.orc_signed_distance_field(_ptr(flags), C.c_int(searchRad), _ptr(dst), C.byref(d))
        return dst

    def normalizePressureMean(self, p, flags, is3D):
        assert p.dtype == np.float32 and p.flags.c_contiguous
        flags = _f32(flags)
        d = _dims(flags, is3D)
        self.lib.orc_normalize_pressure_mean(_ptr(p), _ptr(flags), C.byref(d))
        return p

    def calcLineTrace(self, pos, delta, flags, is3D=True):
        flags = _f32(flags)
        d = _dims(flags, is3D)
        p = _f32(np.asarray(pos, np.float32))
        dl = _f32(np.asarray(delta, np.float32))
        out = np.zeros(3, np.float32)
        hit = self.lib.orc_calc_line_trace(_ptr(p), _ptr(dl), _ptr(flags), C.byref(d), _ptr(out))
        return bool(hit), out

    # -- Lua-side pieces -----------------------------------------------------------------
    def applyBC(self, x, invMask, bc):
        invMask, bc = _f32(invMask), _f32(bc)
        self.lib.orc_apply_bc(_ptr(x), _ptr(invMask), _ptr(bc), C.c_long(x.size))

    def clamp(self, x, lo, hi):
        self.lib.orc_clamp(_ptr(x), C.c_float(lo), C.c_float(hi), C.c_long(x.size))

    def getDx(self, flags):
        return 1.0 / max(flags.shape[2], flags.shape[3], flags.shape[4])

    # -- CNN pieces ----------------------------------------------------------------------
    def conv(self, x, w, bias, is3D, relu):
        x, w, bias = _f32(x), _f32(w), _f32(bias)
        b, cin, z, y, xs = x.shape
        cout = w.shape[0]
        ks = w.shape[-1]
        d = _Dims(b, z, y, xs, 1 if is3D else 0)
        out = np.empty((b, cout, z, y, xs), np.float32)
        self.lib.orc_conv(_ptr(x), _ptr(out), _ptr(w), _ptr(bias), C.byref(d), C.c_int(cin),
                          C.c_int(cout), C.c_int(ks), C.c_int(1 if relu else 0))
        return out

    def sampleStd(self, x):
        x = _f32(x)
        return float(self.lib.orc_sample_std(_ptr(x), C.c_long(x.size)))


class _TensorDesc(C.Structure):
    _fields_ = [("data", C.c_void_p), ("ndim", C.c_int32), ("size", C.c_int64 * 5)]


class Reference(Oracle):
    """The reference's own CPU code (float instantiation) through the fake Lua stack.

    Operators the reference has no CPU implementation for (Jacobi,
    generic/tfluids.cc:836-839) and the Lua-side/CNN pieces fall through to the
    restatement in the parent class.
    """
    name = "reference"

    def __init__(self):
        super().__init__()
        if not have_reference():
            raise RuntimeError("oracle/_ref/libtfluids_ref.so not built (needs /root/reference)")
        self.ref = C.CDLL(REF_SO)

    def num_threads(self):
        return int(self.ref.ref_num_threads())

    def _call(self, name, *args):
        n = len(args)
        kinds = (C.c_int * n)()
        nums = (C.c_double * n)()
        tens = (_TensorDesc * n)()
        strs = (C.c_char_p * n)()
        keep = []
        for i, a in enumerate(args):
            if isinstance(a, np.ndarray):
                assert a.flags.c_contiguous
                if a.dtype == np.float32:
                    kinds[i] = 1
                elif a.dtype == np.int32:
                    kinds[i] = 3
                elif a.dtype == np.float64:
                    kinds[i] = 4
                else:
                    raise TypeError(a.dtype)
                tens[i].data = a.ctypes.data
                tens[i].ndim = a.ndim
                for dd in range(a.ndim):
                    tens[i].size[dd] = a.shape[dd]
                keep.append(a)
            elif isinstance(a, str):
                kinds[i] = 2
                strs[i] = a.encode()
            else:
                kinds[i] = 0
                nums[i] = float(a)
        ret = C.c_double(0)
        err = C.create_string_buffer(1024)
        rc = self.ref.ref_call(name.encode(), C.c_int(0), C.c_int(n), kinds, nums, tens, strs,
                               C.byref(ret), err, C.c_int(1024))
        if rc != 0:
            raise RuntimeError("reference %s: %s" % (name, err.value.decode()))
        return ret.value

    def emptyDomain(self, flags, is3D, bnd=1):
        self._call("emptyDomain", flags, is3D, bnd)
        return flags

    def flagsToOccupancy(self, flags):
        flags = _f32(flags)
        occ = np.empty_like(flags)
        self._call("flagsToOccupancy", flags, occ)
        return occ

    def advectScalar(self, dt, s, U, flags, method="maccormackOurs", sampleOutsideFluid=False,
                     maccormackStrength=0.75):
        s, U, flags = _f32(s), _f32(U), _f32(flags)
        dst = np.full_like(s, np.float32(123.0))
        fwd = np.full_like(s, np.float32(123.0))
        bwd = np.full_like(s, np.float32(123.0))
        fpos = np.zeros_like(U)
        bpos = np.zeros_like(U)
        # Positional order: third_party/tfluids.cc:419-440.
        self._call("advectScalar", dt, s, U, flags, fwd, bwd, _is3d(U), method, fpos, bpos, 1,
                   sampleOutsideFluid, maccormackStrength, dst)
        return dst

    def advectVel(self, dt, U, flags, method="maccormackOurs", maccormackStrength=0.75):
        U, flags = _f32(U), _f32(flags)
        dst = np.full_like(U, np.float32(123.0))
        fwd = np.full_like(U, np.float32(123.0))
        bwd = np.full_like(U, np.float32(123.0))
        self._call("advectVel", dt, U, flags, fwd, bwd, _is3d(U), method, 1, maccormackStrength,
                   dst)
        return dst

    def setWallBcsForward(self, U, flags, as_mask_multiply=False):
        flags = _f32(flags)
        if as_mask_multiply:  # tfluids/set_wall_bcs.lua:29-48
            mask = np.ones_like(U)
            self._call("setWallBcsForward", mask, flags, _is3d(U))
            np.multiply(U, mask, out=U)
        else:
            self._call("setWallBcsForward", U, flags, _is3d(U))

    def velocityDivergenceForward(self, U, flags):
        U, flags = _f32(U), _f32(flags)
        div = np.full_like(flags, np.float32(123.0))
        self._call("velocityDivergenceForward", U, flags, div, _is3d(U))
        return div

    def velocityUpdateForward(self, U, flags, p):
        self._call("velocityUpdateForward", U, _f32(flags), _f32(p), _is3d(U))

    def addBuoyancy(self, U, flags, density, gravity, dt):
        g = _f32(np.asarray(gravity, dtype=np.float32).reshape(3))
        strength = np.zeros(3, np.float32)
        self._call("addBuoyancy", U, _f32(flags), _f32(density), g, strength, dt, _is3d(U))

    def addGravity(self, U, flags, gravity, dt):
        g = _f32(np.asarray(gravity, dtype=np.float32).reshape(3))
        self._call("addGravity", U, _f32(flags), g, dt, _is3d(U))

    def vorticityConfinement(self, U, flags, strength):
        b, c, z, y, x = U.shape
        centered = np.zeros_like(U)
        curl = np.zeros((b, 3, z, y, x), np.float32)
        cnorm = np.zeros((b, 1, z, y, x), np.float32)
        force = np.zeros_like(U)
        self._call("vorticityConfinement", U, _f32(flags), strength, centered, curl, cnorm, force,
                   _is3d(U))

    def calcLineTrace(self, pos, delta, flags, is3D=True):
        flags = _f32(flags)
        assert flags.shape[0] == 1
        p = _f32(np.asarray(pos, np.float32))
        dl = _f32(np.asarray(delta, np.float32))
        out = np.zeros(3, np.float32)
        err = C.create_string_buffer(1024)
        hit = self.ref.ref_calc_line_trace(_ptr(p), _ptr(dl), _ptr(flags), C.c_int(flags.shape[2]),
                                           C.c_int(flags.shape[3]), C.c_int(flags.shape[4]),
                                           C.c_int(1 if is3D else 0), _ptr(out), err,
                                           C.c_int(1024))
        if hit < 0:
            raise RuntimeError("reference calcLineTrace: " + err.value.decode())
        return bool(hit), out


    def volumetricUpSamplingNearestForward(self, ratio, x):
        x = _f32(x)
        nb, nf, nz, ny, nx = x.shape
        out = np.empty((nb, nf, nz * ratio, ny * ratio, nx * ratio), np.float32)
        self._call("volumetricUpSamplingNearestForward", ratio, x, out)
        return out

    def rectangularBlur(self, src, blurRad, is3D):
        src = _f32(src)
        dst, tmp = np.empty_like(src), np.empty_like(src)
        self._call("rectangularBlur", src, blurRad, is3D, dst, tmp)
        return dst

    def signedDistanceField(self, flags, searchRad, is3D):
        flags = _f32(flags)
        dst = np.empty_like(flags)
        self._call("signedDistanceField", flags, searchRad, is3D, dst)
        return dst

    def normalizePressureMean(self, p, flags, is3D):
        inds = np.zeros(p.shape[:1] + p.shape[2:], np.int32)
        self._call("normalizePressureMean", p, _f32(flags), is3D, inds)
        return p

    def velocityDivergenceBackward(self, U, flags, gradOutput):
        U = _f32(U)
        gU = np.full_like(U, np.float32(9.0))
        self._call("velocityDivergenceBackward", U, _f32(flags), _f32(gradOutput), _is3d(U), gU)
        return gU

    def velocityUpdateBackward(self, U, flags, p, gradOutput):
        U = _f32(U)
        gp = np.full_like(_f32(flags), np.float32(9.0))
        self._call("velocityUpdateBackward", U, _f32(flags), _f32(p), _f32(gradOutput), _is3d(U), gp)
        return gp

    def volumetricUpSamplingNearestBackward(self, ratio, x, gradOutput):
        x = _f32(x)
        gi = np.full_like(x, np.float32(9.0))
        self._call("volumetricUpSamplingNearestBackward", ratio, x, _f32(gradOutput), gi)
        return gi

    def findConnectedFluidComponents(self, flags, is3D, ibatch=0):
        flags = _f32(flags).copy()
        comp = np.empty(flags.shape[2:], np.int32)
        sizes = np.zeros(comp.size + 1, np.int32)
        err = C.create_string_buffer(1024)
        n = self.ref.ref_find_connected_fluid_components(
            _ptr(flags), C.c_int(flags.shape[0]), C.c_int(flags.shape[2]), C.c_int(flags.shape[3]),
            C.c_int(flags.shape[4]), C.c_int(1 if is3D else 0), C.c_int(ibatch), _ptr(comp), _ptr(sizes),
            C.c_int(sizes.size), err, C.c_int(1024))
        if n < 0:
            raise RuntimeError("reference findConnectedFluidComponents: " + err.value.decode())
        return comp, sizes[:n].copy()


# ----------------------------------------------------------------------------------------
# The loop around the operators (torch/lib/simulate.lua), restated on top of a backend
# (Oracle or Reference); the projection model (torch/lib/model.lua) is oracle/model.py.
# ----------------------------------------------------------------------------------------
def default_mconf(**over):
    """Keys the hot path reads (lib/simulate.lua:188-291; defaults lib/default_conf.lua)."""
    m = dict(dt=0.1, advectionMethod="maccormackOurs", maccormackStrength=0.75,
             buoyancyScale=0.0, gravityScale=0.0, gravity=None, vorticityConfinementAmp=0.0,
             simMethod="convnet", maxIter=None, is3D=True, normalizeInputThreshold=1e-5)
    m.update(over)
    return m


def create_plume_bcs(batch, densityVal, uScale, rad):
    """tfluids.createPlumeBCs, lib/simulate.lua:47-123 (single-channel density)."""
    U = batch["UDiv"]
    b, c, zdim, ydim, xdim = U.shape
    assert b == 1, "Only single batch allowed."
    is3d = c == 3
    UBC = np.zeros_like(U)
    UBCInv = np.ones_like(U)
    dBC = np.zeros_like(batch["density"])
    dBCInv = np.ones_like(batch["density"])
    centerX = xdim // 2
    centerZ = max(zdim // 2, 1)
    plumeRad = math.floor(xdim * rad)
    vec = np.zeros(c, np.float32)
    vec[1] = 1.0
    vec = vec * np.float32(uScale)
    for z in range(1, zdim + 1):
        for y in range(1, 5):
            for x in range(1, xdim + 1):
                dx = centerX - x
                dz = centerZ - z
                if dx * dx + dz * dz <= plumeRad * plumeRad:
                    UBC[0, :, z - 1, y - 1, x - 1] = vec
                    UBCInv[0, :, z - 1, y - 1, x - 1] = 0
                    dBC[0, :, z - 1, y - 1, x - 1] = densityVal[0]
                    dBCInv[0, :, z - 1, y - 1, x - 1] = 0
                else:
                    UBC[0, :, z - 1, y - 1, x - 1] = 0
                    UBCInv[0, :, z - 1, y - 1, x - 1] = 0
    batch["UBC"], batch["UBCInvMask"] = UBC, UBCInv
    batch["densityBC"], batch["densityBCInvMask"] = dBC, dBCInv
    assert is3d or zdim == 1


def _set_const_vals(be, batch, p, U, flags, density):
    """lib/simulate.lua:130-160."""
    if batch.get("pBC") is not None:
        be.applyBC(p, batch["pBCInvMask"], batch["pBC"])
    if batch.get("UBC") is not None:
        be.applyBC(U, batch["UBCInvMask"], batch["UBC"])
    if batch.get("densityBC") is not None and density is not None:
        be.applyBC(density, batch["densityBCInvMask"], batch["densityBC"])


def simulate(be, mconf, batch, model=None, f64=False):
    """tfluids.simulate, lib/simulate.lua:175-327.  batch holds numpy arrays pDiv, UDiv,
    flags, density (+ optional BC arrays) and is updated in place.  f64: the projection network
    in float64 (model_forward)."""
    p, U, flags, density = batch["pDiv"], batch["UDiv"], batch["flags"], batch.get("density")
    dt = mconf["dt"]
    if density is not None:
        density[...] = be.advectScalar(dt, density, U, flags, mconf["advectionMethod"], False,
                                       mconf["maccormackStrength"])
    U[...] = be.advectVel(dt, U, flags, mconf["advectionMethod"], mconf["maccormackStrength"])
    _set_const_vals(be, batch, p, U, flags, density)

    def gravity_vec():
        g = mconf.get("gravity")
        if g is None:
            g = np.array([0, 1, 0], np.float32)
        return np.array(g, np.float32).copy()

    dx = be.getDx(flags)
    if density is not None and mconf["buoyancyScale"] > 0:
        g = gravity_vec() * np.float32(-(dx / 4) * mconf["buoyancyScale"])
        be.addBuoyancy(U, flags, density, g, dt)
    if mconf["gravityScale"] > 0:
        g = gravity_vec() * np.float32((-dx / 4) * mconf["gravityScale"])
        be.addGravity(U, flags, g, dt)
    if mconf["vorticityConfinementAmp"] > 0:
        be.vorticityConfinement(U, flags, dx * mconf["vorticityConfinementAmp"])
    if mconf["simMethod"] != "convnet":
        be.setWallBcsForward(U, flags)
    _set_const_vals(be, batch, p, U, flags, density)
    if mconf["simMethod"] == "convnet":
        # f64 only as a keyword, and only when asked for: a forward put in place of oracle.api.model_forward with
        # the signature (be, model, pDiv, UDiv, flags, threshold) keeps running the float32 step.
        threshold = mconf.get("normalizeInputThreshold", 1e-5)
        pP, UP, _ = (model_forward(be, model, p, U, flags, threshold, f64=True) if f64 else
                     model_forward(be, model, p, U, flags, threshold))
        p[...] = pP
        U[...] = UP
    else:
        div = be.velocityDivergenceForward(U, flags)
        batch["div"] = div
        if mconf["simMethod"] == "jacobi":
            be.solveLinearSystemJacobi(p, flags, div, mconf["is3D"], 0.0,
                                       mconf.get("maxIter") or 100)
        elif mconf["simMethod"] == "pcg":                       # lib/simulate.lua:280-286
            be.solveLinearSystemPCG(p, flags, div, mconf["is3D"], 1e-4, mconf.get("maxIter") or 100, "ic0")
        else:
            raise ValueError("oracle simulate: simMethod %r not available on CPU"
                             % mconf["simMethod"])
        be.velocityUpdateForward(U, flags, p)
    _set_const_vals(be, batch, p, U, flags, density)
    be.clamp(U, -1e6, 1e6)
