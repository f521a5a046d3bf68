"""The long plume run of tests/test_oracle_long_run.py (its calibration, on the CPU) and tests/test_gpu_long_run.py.

A 64^3 plume with the synthetic geometry (sphere + slab), createPlumeBCs, buoyancy and vorticity confinement,
projected by N fixed-count Jacobi solves.  Its strong buoyancy makes the plume accelerate, so the longest advection
trace (max |U| dt, the host-side proxy of the trace the advectVel tile kernel reports) passes through the three
regimes of the library's advection-tile halo choice (tile_halo_choice, tfl_api.cu):
  state 0                        0.200 cells   (halo 1: traces below 0.45 cells)
  first state >= 0.45 cells      CROSS_HALO2   (halo 2: below 1.4 cells)
  first state >= 1.4 cells       CROSS_TWO_KERNEL, and every later state up to N - 1 stays above it, so the
                                 velocity advection spends N - CROSS_TWO_KERNEL calls in the two-kernel regime
                                 (more than the 16 after which it probes the halo-2 kernel again).
The 2-D run is the same scene on a 128^2 grid (no vorticity confinement, as in test_gpu_step.py)."""
import numpy as np

import oracle
from scenes import plume_batch

N = 100
DT = 0.1
CROSS_HALO2 = 10
CROSS_TWO_KERNEL = 59
KEYS = ("pDiv", "UDiv", "density")


def make_batch(is3d):
    """Initial state and BCs: [1][c][64][64][64] in 3-D, [1][c][1][128][128] in 2-D (numpy)."""
    n = 64 if is3d else 128
    return plume_batch(n, is3d, amp=2.0, inflow=n / 128.0 * 4)


def make_mconf(is3d, sim_method="jacobi"):
    return oracle.default_mconf(dt=DT, maccormackStrength=0.6, buoyancyScale=16.0,
                                vorticityConfinementAmp=3.0 if is3d else 0.0, simMethod=sim_method, maxIter=30,
                                is3D=is3d)


def trace_proxy(U):
    """Longest trace of a velocity field in cells, max |U| dt."""
    return float(np.abs(U).max()) * DT


def oracle_trajectory(orc, is3d, steps=N):
    """(batch, states): states[s] holds copies of pDiv, UDiv and density after s oracle steps (states[0] is the
    initial state); batch holds the flags and BCs."""
    batch = make_batch(is3d)
    mconf = make_mconf(is3d)
    states = [{k: batch[k].copy() for k in KEYS}]
    work = {k: v.copy() for k, v in batch.items()}
    for _ in range(steps):
        oracle.simulate(orc, mconf, work, None)
        states.append({k: work[k].copy() for k in KEYS})
    return batch, states
