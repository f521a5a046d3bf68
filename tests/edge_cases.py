"""The smallest legal grids and strongly non-cubic ones, with the inputs both edge-size files use: the oracle pinned
on the compiled reference (test_oracle_edge_sizes.py, CPU) and the library against the oracle
(test_gpu_edge_sizes.py).  Both draw their fields from fields() here, so the GPU file runs exactly the inputs the
oracle is pinned on."""
import numpy as np

from fluidnet_b200 import synth

DT = 0.3
STRENGTH = 0.75
TRACES = (0.2, 1.0, 3.0, 20.0)   # longest trace of each velocity field, in cells (max|U| * DT)

# (nx, ny, nz); nz == 1 is a 2-D grid.  What each one reaches on the GPU is in test_gpu_edge_sizes.ROWS.
GRIDS = [
    (3, 3, 3), (4, 3, 3), (4, 3, 5), (33, 3, 3), (3, 17, 4), (36, 3, 3), (4, 17, 4), (1028, 3, 3),
    (4, 300, 3), (4, 3, 300), (128, 8, 4), (128, 8, 5), (128, 24, 4), (256, 8, 4), (128, 8, 8),
    (3, 3, 1), (5, 3, 1), (3, 41, 1), (4, 3, 1), (1028, 3, 1), (3, 600, 1),
]


def traces(shape):
    """The trace lengths run on this grid.  On the rows of 300 cells and more, random 3- and 20-cell traces along
    the long axis end where the line trace finds no fluid cell to back off to: the reference raises there ("Cannot
    find non-geometry point"), the oracle counts a trace fault, and neither is a valid input."""
    return TRACES if max(shape) < 300 else TRACES[:2]


def batches(shape):
    return (1, 2, 3) if shape[2] == 1 else (1, 2)


CASES = [(s, nb) for s in GRIDS for nb in batches(s)]
CASE_IDS = ["%dx%dx%d-nb%d" % (s + (nb,)) for s, nb in CASES]


GRAVITY = [0.2, -0.5, 0.1]
UP_RATIOS = (1, 2, 3)


def pointwise_ops(fl, s, p):
    """(name, fn(backend, U)) for the operators that update U in place."""
    return (
        ("setWallBcs", lambda be, u: be.setWallBcsForward(u, fl)),
        ("velocityUpdate", lambda be, u: be.velocityUpdateForward(u, fl, p)),
        ("addBuoyancy", lambda be, u: be.addBuoyancy(u, fl, s, GRAVITY, 0.1)),
        ("addGravity", lambda be, u: be.addGravity(u, fl, GRAVITY, 0.1)),
        ("vorticityConfinement", lambda be, u: be.vorticityConfinement(u, fl, 0.4)),
    )


def empty_domain_bnds(shape):
    """Border widths emptyDomain accepts on this grid (init.lua:549-551: every extent >= 2 bnd + 1)."""
    ext = shape if shape[2] > 1 else shape[:2]
    return [b for b in (1, 2) if min(ext) >= 2 * b + 1]


def blur_radii(shape):
    return (1, 2, max(shape) + 1)


def fields(shape, nb, trace=1.0, seed=0):
    """flags (an empty box: on these cross-sections the synth sphere fills whole stretches of the interior, where
    the reference's line trace gives up, "Cannot find non-geometry point"), U with longest trace `trace` cells at DT
    (wall BCs not yet applied), a scalar s in [0, 1) and p in [-0.5, 0.5)."""
    nx, ny, nz = shape
    is3d = nz > 1
    flags = synth.make_flags(nx, ny, nz, is3d, nb=nb, geometry=False)
    rng = np.random.default_rng(seed)
    U = rng.standard_normal((nb, 3 if is3d else 2, nz, ny, nx))
    U = np.ascontiguousarray((U * (trace / (DT * np.abs(U).max()))).astype(np.float32))
    s = rng.random(flags.shape).astype(np.float32)
    p = (rng.random(flags.shape) - 0.5).astype(np.float32)
    return flags, U, s, p
