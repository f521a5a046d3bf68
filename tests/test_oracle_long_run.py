"""Calibration of the long plume run (tests/long_run.py) on the oracle alone: the longest trace starts below the
halo-1 limit, crosses 0.45 and 1.4 cells at the recorded steps and stays above 1.4 cells to the end, so the GPU
long-run module keeps driving every regime of the advection-tile halo choice.  About 8 s of oracle time at 64^3
(0.065 s per step on 8 cores)."""
import long_run


def test_trajectory_crosses_every_tile_halo_regime(orc):
    orc.lib.orc_reset_trace_faults()
    _, states = long_run.oracle_trajectory(orc, True)
    tr = [long_run.trace_proxy(s["UDiv"]) for s in states[:long_run.N]]
    assert tr[0] < 0.45, "the initial state's trace is %.3f cells, not below 0.45" % tr[0]
    first_045 = next(s for s, t in enumerate(tr) if t >= 0.45)
    first_14 = next((s for s, t in enumerate(tr) if t >= 1.4), None)
    assert first_045 == long_run.CROSS_HALO2, \
        "the trace crosses 0.45 cells at step %d, not at step %d" % (first_045, long_run.CROSS_HALO2)
    assert first_14 == long_run.CROSS_TWO_KERNEL, \
        "the trace crosses 1.4 cells at step %s, not at step %d" % (first_14, long_run.CROSS_TWO_KERNEL)
    below = [s for s in range(first_14, long_run.N) if tr[s] < 1.4]
    assert not below, "the trace drops below 1.4 cells again at steps %s" % below
    assert long_run.N - first_14 >= 20
    assert orc.trace_faults() == 0


def test_2d_trajectory_stays_in_the_domain(orc):
    """The 2-D run of the GPU module: N steps without a trace leaving the domain, and a plume that accelerates."""
    orc.lib.orc_reset_trace_faults()
    _, states = long_run.oracle_trajectory(orc, False)
    assert orc.trace_faults() == 0
    assert long_run.trace_proxy(states[-1]["UDiv"]) > 2 * long_run.trace_proxy(states[0]["UDiv"])
