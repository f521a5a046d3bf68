"""What the GPU tests build their cases from: the plume scene and its step configuration, the upload of a numpy
batch, the bank tables and batch-normalized models of synth.make_model, and the max-relative comparison."""
import numpy as np
import torch

import oracle
from fluidnet_b200 import synth


def plume_batch(shape, is3d=True, nb=1, geometry=True, flags_seed=7, uniform=False, amp=3.0, seed=1234, inflow=None):
    """The numpy batch {pDiv (zeros), UDiv, flags, density} of synth's flags with the wall BCs set on a smooth (or,
    uniform=True, uniform random) velocity of amplitude amp.  shape: a cube edge n (an n x n grid in 2-D) or
    (nz, ny, nx).  inflow: the speed scale of the plume's inflow (createPlumeBCs with density 1 and radius 0.15:
    UBC, UBCInvMask, densityBC, densityBCInvMask); None adds no BCs."""
    nz, ny, nx = shape if isinstance(shape, tuple) else ((shape if is3d else 1), shape, shape)
    flags = synth.make_flags(nx, ny, nz, is3d, nb=nb, geometry=geometry, seed=flags_seed)
    U = (synth.make_velocity if uniform else synth.make_smooth_velocity)(flags, is3d, amp=amp, seed=seed)
    oracle.Oracle().setWallBcsForward(U, flags)
    batch = {"pDiv": np.zeros_like(flags), "UDiv": U, "flags": flags, "density": synth.make_density(flags)}
    if inflow is not None:
        oracle.create_plume_bcs(batch, [1.0], inflow, 0.15)
    return batch


def step_mconf(n, **over):
    """The plume step on an n-wide grid: maccormackOurs at strength 0.6, buoyancy 2 n / 128, vorticity confinement
    3, the convnet projection; `over` replaces or adds keys."""
    return oracle.default_mconf(**dict(dict(dt=0.1, maccormackStrength=0.6, buoyancyScale=2.0 * n / 128,
                                            vorticityConfinementAmp=3.0, simMethod="convnet"), **over))


def to_gpu(batch):
    return {k: torch.from_numpy(v.copy()).cuda() for k, v in batch.items() if v is not None}


def inputs_of(batch, seed=77):
    """(p0, network inputs on the GPU): a small signed pDiv of the batch's shape, and (p0, UDiv, flags)."""
    p0 = (synth.make_density(batch["flags"], seed=seed) - np.float32(0.5)) * np.float32(0.1)
    return p0, tuple(torch.from_numpy(a).cuda() for a in (p0, batch["UDiv"], batch["flags"]))


def banks(num, agg, kind=None, s=1, j=3):
    """A banks table of synth.make_model (split at stage s, joined at stage j); "type" is set only when kind is
    given, as a banksType read from a reference file would be."""
    bk = {"num": num, "split_stage": s, "join_stage": j, "aggregate": agg}
    if kind is not None:
        bk["type"] = kind
    return bk


def bn_model(train, is3d=True, model_type="default", bk=None, inputs=None, relu6=False, affine=True):
    """synth.make_model with batch normalization on batch (train) or running statistics (train=None: none); relu6
    sets nonlinType 'relu6' and scales the first convolution by 30, so the first stage's values cross 6."""
    m = synth.make_model(is3d, model_type=model_type, banks=bk, inputs=inputs,
                         batch_norm=None if train is None else {"train": train, "affine": affine})
    if relu6:
        m["nonlinType"] = "relu6"
        first = m["layers"][0] if not isinstance(m["layers"][0], list) else m["layers"][0][0]
        first[0][...] *= np.float32(30.0)
    return m


def close(got, want, tol, what):
    """|got - want| <= tol * max|want| (max|want| at least 1e-6)."""
    err = np.abs(got.astype(np.float64) - want.astype(np.float64)).max()
    scale = max(np.abs(want).max(), 1e-6)
    assert err <= tol * scale, "%s: max err %g vs scale %g" % (what, err, scale)


def write_binvox(path, dims, occ_flat):
    """A .binvox file whose run-length body decodes, through the reference parser's quirks (formats.load_binvox), to
    occ_flat: one (value, 1) pair per cell -- a run writes count + 1 = 2 cells and moves on by 1, so the next run
    overwrites the second -- and a final pair the parser drops.  The last cell keeps the value of the one before it
    (the parser stops there), so occ_flat must end with two equal values."""
    assert occ_flat[-1] == occ_flat[-2]
    body = bytearray()
    for v in occ_flat:
        body += bytes([int(v), 1])
    body += bytes([0, 0])
    head = "#binvox 1\ndim %d %d %d\ntranslate 0 0 0\nscale 1\ndata\n" % tuple(dims)
    with open(path, "wb") as f:
        f.write(head.encode("ascii") + bytes(body))


def fields_with_random_p(nz, ny, nx, is3d=True):
    import oracle
    from fluidnet_b200 import synth
    flags = synth.make_flags(nx, ny, nz, is3d, nb=1, geometry=True)
    U = synth.make_smooth_velocity(flags, is3d, amp=3.0)
    oracle.Oracle().setWallBcsForward(U, flags)
    p = (np.random.RandomState(5).rand(*flags.shape).astype(np.float32) - 0.5)
    return {"pDiv": p, "UDiv": U, "flags": flags, "density": synth.make_density(flags)}
