"""The divergence statistics of torch/lib/calc_stats.lua:81-123 after every step, taken behind the running step
(tfl_monitor_*, include/tfl.h; DESIGN.md section 6b).

For each batch entry a record holds div_norm = sqrt(sum d^2) (the reference's `div[i]:norm()`), div_max = max |d| and
u_max = max |U|, d being what tfluids.velocityDivergenceForward writes.  `record` enqueues a device reduction on the
current stream and never waits; the record lands in pinned host memory and `take` / `drain` collect it later.

    mon = StepMonitor(None, batch, capacity=64)
    for i in range(n):
        step()
        mon.record(batch)                   # refused when `capacity` records are waiting: take some first
        rows += mon.drain()                 # the records that have landed, oldest first
    rows += mon.drain(wait=True)

On z-slabs, `NativeSlabSimulator.monitor()` returns a SlabStepMonitor: each rank reduces its own planes and keeps one
partial per plane, and `combine_planes` adds every rank's partials in ascending global z -- the device's own last
step, so the totals equal the whole-grid monitor's bit for bit whatever the number of ranks.
"""
import ctypes as C
import math

import numpy as np

from . import tfluids
from ._lib import TflError


def _nanmax(a, b):
    """max that propagates NaN, as the device's reduction does."""
    return b if (b > a or b != b) else a


def combine_planes(parts):
    """Totals [nb][3] = (div_norm, div_max, u_max) from per-plane partials: `parts` is a list of (z0, partials) with
    partials [nb][planes][3] = (sum d^2, max |d|, max |U|) of global planes z0, z0 + 1, ... (one entry per rank, any
    order).  The planes must tile [0, gnz) without gaps or overlaps.  Sums run in ascending global z from 0 in fp64,
    then the square root -- what k_monitor_finish does for a whole grid."""
    parts = sorted(((int(z0), np.asarray(p, np.float64)) for z0, p in parts), key=lambda zp: zp[0])
    z = 0
    for z0, p in parts:
        if p.ndim != 3 or p.shape[2] != 3 or p.shape[0] != parts[0][1].shape[0]:
            raise ValueError("combine_planes: partials must be [nb][planes][3] with one nb, got %r" % (p.shape,))
        if z0 != z:
            raise ValueError("combine_planes: planes [%d, %d) are missing or given twice" % (min(z, z0), max(z, z0)))
        z = z0 + p.shape[1]
    planes = np.concatenate([p for _, p in parts], axis=1)
    out = np.empty((planes.shape[0], 3), np.float64)
    for b in range(planes.shape[0]):
        s, dm, um = 0.0, 0.0, 0.0
        for q in planes[b].tolist():           # Python floats: one IEEE double addition at a time, in order
            s += q[0]
            dm = _nanmax(dm, q[1])
            um = _nanmax(um, q[2])
        out[b] = (math.sqrt(s), dm, um)
    return out


class StepMonitor:
    """A ring of `capacity` records of the fields of `batch` (its 'UDiv' and 'flags', [nb][c][gnz][ny][nx] CUDA
    float32).  ctx: a tfluids.Context, or None for the context of the batch's device."""

    def __init__(self, ctx, batch, capacity=64):
        flags = batch["flags"]
        self.ctx = ctx if ctx is not None else tfluids.context(flags.device)
        self.nb, self.gnz = int(flags.size(0)), int(flags.size(2))
        self._open(capacity)

    def _open(self, capacity):
        self.capacity = int(capacity)
        self.pending = 0                                   # recorded, not yet taken
        self._buf = (C.c_double * (self.nb * self.gnz * 3))()
        h = C.c_void_p()
        self.ctx.check(self.ctx.lib.tfl_monitor_create(self.ctx.h, self.nb, self.gnz, self.capacity, C.byref(h)))
        self.h = h

    @property
    def full(self):
        return self.pending == self.capacity

    def record(self, batch):
        """Enqueue the reduction of batch['UDiv'] and batch['flags'] on the current stream; returns the record's
        index.  Never waits."""
        U, flags = batch["UDiv"], batch["flags"]
        if tfluids._ctx_for(flags) is not self.ctx:
            raise TflError("StepMonitor: the batch lives on another device than the monitor")
        assert U.is_contiguous() and flags.is_contiguous(), "StepMonitor: contiguous 5-D tensors are needed"
        idx = C.c_int64(-1)
        self.ctx.check(self.ctx.lib.tfl_monitor_record(self.ctx.h, self.h, tfluids._grid(U), tfluids._grid(flags),
                                                       C.byref(idx)))
        self.pending += 1
        return idx.value

    def _take(self, wait):
        """-> None, or (index, z0, planes, values): values [nb][3] totals (planes == 0) or [nb][planes][3] partials."""
        idx, z0, n = C.c_int64(-1), C.c_int32(0), C.c_int32(0)
        self.ctx.check(self.ctx.lib.tfl_monitor_take(self.ctx.h, self.h, 1 if wait else 0, C.byref(idx), self._buf,
                                                     C.byref(z0), C.byref(n)))
        if idx.value < 0:
            return None
        self.pending -= 1
        shape = (self.nb, n.value, 3) if n.value else (self.nb, 3)
        vals = np.frombuffer(self._buf, np.float64, int(np.prod(shape))).reshape(shape).copy()
        return idx.value, z0.value, n.value, vals

    def take(self, wait=True):
        """-> (index, [nb][3] float64 array of div_norm, div_max, u_max) of the oldest record, or None if wait is
        false and it has not landed.  Raises when no record is waiting."""
        got = self._take(wait)
        return None if got is None else (got[0], got[3])

    def drain(self, wait=False):
        """Every waiting record that has landed (with wait, all of them), oldest first: [(index, values), ...]."""
        out = []
        while self.pending:
            got = self.take(wait)
            if got is None:
                break
            out.append(got)
        return out

    def close(self):
        """Wait for the records in flight and free the monitor."""
        if getattr(self, "h", None):
            self.ctx.lib.tfl_monitor_destroy(self.ctx.h, self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


class SlabStepMonitor(StepMonitor):
    """The monitor of a NativeSlabSimulator (`sim.monitor()`): `record` is collective like a step (it refreshes the
    ghost plane the divergence reads above the owned planes, tfl_slab_sim_monitor_record); each rank's records hold the
    partials of its owned planes.

    Over a run, `record_frame` after every step records and, when the ring is full, moves this rank's oldest record
    (long landed) into a host list -- no collective, so no rank waits for the others or for its stream.  `collect`
    after the run gathers every rank's list once and combines it: every rank gets the whole grid's records.  `take` is
    the same for one record at a time; it is collective, and through torch.distributed an object gather waits for the
    current stream, so use it where a synchronised step costs nothing (tests, end of run)."""

    def __init__(self, sim, capacity=64):
        self.sim, self.ctx = sim, sim.ctx
        self.nb, self.gnz = 1, int(sim._shape[2])
        self.kept = []                    # (index, z0, partials) of this rank taken by record_frame
        self._open(capacity)

    def record(self, batch=None):
        """Collective: enqueue this rank's record of the simulator's fields on the current stream; never waits."""
        self.ctx.use_current_stream()
        idx = C.c_int64(-1)
        self.ctx.check(self.ctx.lib.tfl_slab_sim_monitor_record(self.ctx.h, self.sim.h, self.h, C.byref(idx)))
        self.pending += 1
        return idx.value

    def take_partials(self, wait=True):
        """-> (index, z0, [1][planes][3] partials of global planes z0 ..) of this rank's oldest record, or None."""
        got = self._take(wait)
        return None if got is None else (got[0], got[1], got[3])

    def record_frame(self):
        """Collective like `record`: record this step, after keeping this rank's oldest record if the ring is full."""
        if self.full:
            self.kept.append(self.take_partials(True))
        return self.record()

    def _allgather(self, obj):
        if self.sim._allgather is not None:
            return self.sim._allgather(obj)
        if self.sim.world == 1:
            return [obj]
        import torch.distributed as dist
        out = [None] * self.sim.world
        dist.all_gather_object(out, obj, group=self.sim.group)
        return out

    @staticmethod
    def _combine(per_rank):
        """per_rank: every rank's list of (index, z0, partials), in record order -> [(index, [1][3] totals), ...]."""
        n = {len(x) for x in per_rank}
        idx = [[r[0] for r in x] for x in per_rank]
        if len(n) != 1 or any(i != idx[0] for i in idx):
            raise TflError("SlabStepMonitor: the ranks hold records %s; every rank must record alike"
                           % [(i[0], i[-1], len(i)) if i else () for i in idx])
        return [(recs[0][0], combine_planes([(r[1], r[2]) for r in recs])) for recs in zip(*per_rank)]

    def collect(self):
        """Collective: every record kept by `record_frame` and every one still in the ring (waiting for them), combined
        over the ranks with one gather."""
        while self.pending:
            self.kept.append(self.take_partials(True))
        mine, self.kept = self.kept, []
        return self._combine(self._allgather(mine))

    def take(self, wait=True):
        """Collective: (index, [1][3] totals) of the oldest record, combined over every rank (waits for it)."""
        return self._combine(self._allgather([self.take_partials(True)]))[0]

    def drain(self, wait=True):
        """Collective: every waiting record, combined (waits for each)."""
        return [self.take() for _ in range(self.pending)]
