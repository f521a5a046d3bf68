"""Seeded input cases shared by the CPU (oracle) and GPU (libtfl) parity tests."""
import numpy as np

from fluidnet_b200 import synth

import ref_record

# (name, is3d, (nx, ny, nz), geometry, exotic flags, velocity amplitude, smooth velocity)
CASES = [
    ("3d_empty", True, (20, 18, 16), False, False, 2.0, False),
    ("3d_geom", True, (24, 20, 16), True, False, 2.0, False),
    ("3d_geom_fast", True, (24, 20, 16), True, False, 25.0, False),
    ("3d_exotic", True, (20, 20, 14), True, True, 6.0, True),
    ("2d_empty", False, (40, 36, 1), False, False, 2.0, False),
    ("2d_geom_fast", False, (40, 36, 1), True, False, 25.0, True),
    ("2d_exotic", False, (33, 29, 1), True, True, 6.0, False),
]
CASE_IDS = [c[0] for c in CASES]


def build(case, nb=2):
    name, is3d, (nx, ny, nz), geom, exotic, amp, smooth = case
    flags = synth.make_flags(nx, ny, nz, is3d, nb=nb, geometry=geom, exotic=exotic)
    mk = synth.make_smooth_velocity if smooth else synth.make_velocity
    U = mk(flags, is3d, amp=amp)
    dens = synth.make_density(flags)
    p = synth.make_density(flags, seed=99) - np.float32(0.5)
    return dict(name=name, is3d=is3d, flags=flags, U=U, density=dens, p=np.ascontiguousarray(p))


def bits_equal(a, b):
    a, b = ref_record.expected(a), ref_record.expected(b)
    if isinstance(a, ref_record.Recorded):
        a, b = b, a
    if isinstance(b, ref_record.Recorded):
        return b.matches(a)
    a = np.ascontiguousarray(a, np.float32)
    b = np.ascontiguousarray(b, np.float32)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def describe_diff(a, b):
    if any(isinstance(ref_record.expected(x), ref_record.Recorded) for x in (a, b)):
        return "differs from the recorded reference output (tests/golden/ref_calls.json.gz)"
    d = np.abs(a.astype(np.float64) - b.astype(np.float64))
    bad = int((a.view(np.uint32) != b.view(np.uint32)).sum())
    return "max|diff|=%g, %d of %d cells differ in bits" % (d.max(), bad, a.size)
