"""Adapter giving the product (fluidnet_b200 -> libtfl.so through the C ABI) the same
numpy-level API as oracle.Oracle, so GPU parity tests read like the oracle tests."""
import numpy as np
import torch

from fluidnet_b200 import tfluids


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()


def host(t):
    return np.ascontiguousarray(t.detach().cpu().numpy())


class GpuBackend:
    name = "libtfl"

    def trace_faults(self):
        return tfluids.context().trace_faults()

    def emptyDomain(self, flags, is3D, bnd=1):
        t = dev(flags)
        tfluids.emptyDomain(t, is3D, bnd)
        flags[...] = host(t)
        return flags

    def flagsToOccupancy(self, flags):
        t = dev(flags)
        o = torch.full_like(t, 55.0)
        tfluids.flagsToOccupancy(t, o)
        return host(o)

    def advectScalar(self, dt, s, U, flags, method="maccormackOurs", sampleOutsideFluid=False,
                     maccormackStrength=0.75, in_place=False):
        ts, tU, tf = dev(s), dev(U), dev(flags)
        if in_place:
            tfluids.advectScalar(dt, ts, tU, tf, method, None, sampleOutsideFluid, maccormackStrength)
            return host(ts)
        d = torch.full_like(ts, 123.0)
        tfluids.advectScalar(dt, ts, tU, tf, method, d, sampleOutsideFluid, maccormackStrength)
        assert torch.equal(ts, dev(s)), "advectScalar modified its input"
        return host(d)

    def advectVel(self, dt, U, flags, method="maccormackOurs", maccormackStrength=0.75, in_place=False):
        tU, tf = dev(U), dev(flags)
        if in_place:
            tfluids.advectVel(dt, tU, tf, method, None, maccormackStrength)
            return host(tU)
        d = torch.full_like(tU, 123.0)
        tfluids.advectVel(dt, tU, tf, method, d, maccormackStrength)
        return host(d)

    def setWallBcsForward(self, U, flags, as_mask_multiply=False):
        tf = dev(flags)
        if as_mask_multiply:           # what tfluids.SetWallBcs does (set_wall_bcs.lua:29-48)
            mask = torch.ones_like(dev(U))
            tfluids.setWallBcsForward(mask, tf)
            U[...] = host(dev(U) * mask)
        else:
            t = dev(U)
            tfluids.setWallBcsForward(t, tf)
            U[...] = host(t)

    def velocityDivergenceForward(self, U, flags):
        tU, tf = dev(U), dev(flags)
        d = torch.full_like(tf, 123.0)
        tfluids.velocityDivergenceForward(tU, tf, d)
        return host(d)

    def velocityUpdateForward(self, U, flags, p):
        t = dev(U)
        tfluids.velocityUpdateForward(t, dev(flags), dev(p))
        U[...] = host(t)

    def addBuoyancy(self, U, flags, density, gravity, dt):
        t = dev(U)
        tfluids.addBuoyancy(t, dev(flags), dev(density), torch.tensor(gravity, dtype=torch.float32), dt)
        U[...] = host(t)

    def addGravity(self, U, flags, gravity, dt):
        t = dev(U)
        tfluids.addGravity(t, dev(flags), torch.tensor(gravity, dtype=torch.float32), dt)
        U[...] = host(t)

    def vorticityConfinement(self, U, flags, strength):
        t = dev(U)
        tfluids.vorticityConfinement(t, dev(flags), strength)
        U[...] = host(t)

    def solveLinearSystemJacobi(self, p, flags, div, is3D, pTol=1e-5, maxIter=1000):
        t = dev(p)
        r = tfluids.solveLinearSystemJacobi(t, dev(flags), dev(div), is3D, pTol, maxIter)
        self.last_jacobi_iters = tfluids.solveLinearSystemJacobi.last_iterations
        p[...] = host(t)
        return r

    def solveLinearSystemPCG(self, p, flags, div, is3D, tol=1e-6, maxIter=1000, precondType="ic0"):
        t = dev(p)
        r = tfluids.solveLinearSystemPCG(t, dev(flags), dev(div), is3D, tol, maxIter, precondType)
        self.last_pcg_iters = tfluids.solveLinearSystemPCG.last_iterations
        p[...] = host(t)
        return r

    def applyBC(self, x, invMask, bc):
        t = dev(x)
        tfluids.applyBC(t, dev(invMask), dev(bc))
        x[...] = host(t)

    def clamp(self, x, lo, hi):
        t = dev(x)
        tfluids.clamp(t, lo, hi)
        x[...] = host(t)

