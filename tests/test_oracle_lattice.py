"""The oracle (oracle/tfluids_oracle.c) against the reference's compiled CPU code, bit for bit, on lattice advection
inputs (tests/lattice_cases.py): traces that end exactly on cell centres, faces, the domain ends and the faces of
solids, and trace lengths exactly at, and one or two ulps around, the branch thresholds of the trace loop and of the
GPU's clear-space fast paths.  Random inputs (tests/test_oracle_vs_ref.py) essentially never land there."""
import numpy as np
import pytest

import lattice_cases as L
import oracle
from cases import bits_equal, describe_diff

METHODS = list(oracle.ADVECT_METHODS)


@pytest.fixture(scope="module")
def fields(orc):
    return {c[0]: L.build(c, nb=2, wall_bcs=orc.setWallBcsForward) for c in L.FIELD_CASES}


def test_census_reaches_every_tie(fields):
    """The inputs keep hitting the boundaries they are built for (minimum counts over the cases, per dimension)."""
    for is3d in (True, False):
        tot = {}
        for c in L.FIELD_CASES:
            if c[1] != is3d:
                continue
            f = fields[c[0]]
            for k, v in L.tie_census(f["flags"], f["U"], f["dt"]).items():
                tot[k] = tot.get(k, 0) + v
        need = dict(centre=500, face=500, domain_end=20, solid_face=10, reach=20, reach_fluid=20)
        if is3d:
            need.update(halo1=100, halo2=100, step0=1, step1=50, step2=20)
        for k, n in need.items():
            assert tot[k] >= n, "%s: %d traces at %s, want >= %d (census %s)" % ("3-D" if is3d else "2-D", tot[k], k,
                                                                                 n, tot)


@pytest.mark.parametrize("case", L.FIELD_CASES, ids=L.FIELD_IDS)
def test_advect_scalar(orc, ref, fields, case):
    f = fields[case[0]]
    for method in METHODS:
        for outside in (False, True):
            a = orc.advectScalar(f["dt"], f["density"], f["U"], f["flags"], method, outside, 0.6)
            b = ref.advectScalar(f["dt"], f["density"], f["U"], f["flags"], method, outside, 0.6)
            assert bits_equal(a, b), "%s outside=%s: %s" % (method, outside, describe_diff(a, b))
    assert orc.trace_faults() == 0


@pytest.mark.parametrize("case", L.FIELD_CASES, ids=L.FIELD_IDS)
def test_advect_vel(orc, ref, fields, case):
    f = fields[case[0]]
    for method in METHODS:
        a = orc.advectVel(f["dt"], f["U"], f["flags"], method, 0.6)
        b = ref.advectVel(f["dt"], f["U"], f["flags"], method, 0.6)
        assert bits_equal(a, b), "%s: %s" % (method, describe_diff(a, b))
    assert orc.trace_faults() == 0


@pytest.mark.parametrize("kind", ["box", "open", "geom", "exotic"])
@pytest.mark.parametrize("is3d", [True, False], ids=["3d", "2d"])
def test_line_trace_on_the_lattice(orc, ref, kind, is3d):
    """calcLineTrace from cell centres near solids and the domain ends, axis-aligned deltas of 0.25 k cells.  Where
    the reference raises, the oracle must count a trace fault (deviation (1) of DESIGN.md section 1)."""
    flags = L.make_flags(kind, is3d)
    n = raised = 0
    for pos, delta in L.trace_starts(flags, is3d):
        before = orc.trace_faults()
        ha, pa = orc.calcLineTrace(pos, delta, flags, is3d)
        try:
            hb, pb = ref.calcLineTrace(pos, delta, flags, is3d)
        except RuntimeError:
            raised += 1
            assert orc.trace_faults() > before, (pos, delta, "the reference raised, the oracle counted no fault")
            continue
        assert orc.trace_faults() == before, (pos, delta, "the oracle counted a fault, the reference did not raise")
        assert ha == hb and bits_equal(pa, pb), (pos, delta, pa, pb)
        n += 1
    assert n >= 500
