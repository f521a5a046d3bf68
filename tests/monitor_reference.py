"""The step monitor's reduction restated on the host (tfl_monitor.cu): the same fp64 additions in the same order, so
the results must equal the device's bit for bit.  d comes from the oracle's velocityDivergenceForward."""
import math

import numpy as np

THREADS = 256
CHUNKS = 8


def _chunk_sum(d2):
    """One CTA of k_monitor_chunks: thread t adds cells t, t + 256, ... in order; each warp's lanes reduce with
    shfl_down by 16, 8, 4, 2, 1; thread 0 adds the eight warp sums in order."""
    n = -(-d2.size // THREADS) * THREADS
    cells = np.zeros(n, np.float64)
    cells[:d2.size] = d2                     # adding 0.0 to a sum of squares changes nothing
    s = np.zeros(THREADS, np.float64)
    for row in cells.reshape(-1, THREADS):
        s = s + row
    w = s.reshape(THREADS // 32, 32)
    for off in (16, 8, 4, 2, 1):
        nxt = w.copy()
        nxt[:, :32 - off] = w[:, :32 - off] + w[:, off:]
        w = nxt
    total = 0.0
    for v in w[:, 0].tolist():
        total += v
    return total


def plane_partials(div, U):
    """[nb][nz][3] = (sum d^2, max |d|, max |U|) per plane, with the device's split of a plane into row chunks."""
    nb, _, nz, ny, nx = div.shape
    chunks = min(ny, CHUNKS)
    out = np.zeros((nb, nz, 3), np.float64)
    d2 = div.astype(np.float64) ** 2
    for b in range(nb):
        for z in range(nz):
            s = 0.0
            for c in range(chunks):
                r0, r1 = c * ny // chunks, (c + 1) * ny // chunks
                s += _chunk_sum(d2[b, 0, z, r0:r1].ravel())
            out[b, z] = (s, float(np.abs(div[b, 0, z]).max()), float(np.abs(U[b, :, z]).max()))
    return out


def totals(planes):
    """[nb][3] = (div_norm, div_max, u_max): planes added in ascending z from 0, then the square root."""
    out = np.zeros((planes.shape[0], 3), np.float64)
    for b in range(planes.shape[0]):
        s = 0.0
        for v in planes[b, :, 0].tolist():
            s += v
        out[b] = (math.sqrt(s), planes[b, :, 1].max(), planes[b, :, 2].max())
    return out


def record(orc, U, flags):
    """The monitor's record of host fields (U [nb][c][z][y][x], flags [nb][1][z][y][x])."""
    div = orc.velocityDivergenceForward(U, flags)
    return totals(plane_partials(div, U))
