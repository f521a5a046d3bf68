"""Density frames to disk behind the running step (tfl_recorder_*, include/tfl.h).

The demo's save branch (torch/fluid_net_3d_sim.lua:286-290) permutes the density to x-slowest order, copies it to the
host synchronously and appends it to a `.vbox` file.  `FrameRecorder` does the same without stalling the stream:
`capture` enqueues a pack kernel (the permutation) on the current stream and a copy into a ring of pinned host frames
on a stream of its own; `take` hands the oldest frame over once its copy has landed; `release` gives its slot back.

    rec = FrameRecorder((nz, ny, nx))
    with formats.VboxWriter(path, (nx, ny, nz), num_frames) as w:
        for i in range(num_frames):
            step()
            if i % 3 == 2:
                rec.record(density, w)        # waits only when every slot holds an unwritten frame
            rec.drain(w)                      # writes the frames whose copies have landed
        rec.drain(w, wait=True)
    rec.close()
"""
import ctypes as C

import numpy as np

from . import _lib, tfluids
from ._lib import TflError


class FrameRecorder:
    def __init__(self, shape, slots=3, device=None):
        """shape: (nz, ny, nx) or the grid's (1, 1, nz, ny, nx); slots: pinned host frames in the ring."""
        shape = tuple(int(v) for v in shape)
        if len(shape) == 5:
            if shape[:2] != (1, 1):
                raise TflError("FrameRecorder: a recorder takes a [1][1][nz][ny][nx] grid, not %r" % (shape,))
            shape = shape[2:]
        if len(shape) != 3:
            raise TflError("FrameRecorder: shape must be (nz, ny, nx), got %r" % (shape,))
        self.shape = shape
        self.slots = int(slots)
        self.ctx = tfluids.context(device)
        h = C.c_void_p()
        self.ctx.check(self.ctx.lib.tfl_recorder_create(self.ctx.h, shape[0], shape[1], shape[2], self.slots, C.byref(h)))
        self.h = h
        self.captured = 0         # captured, not yet taken
        self.taken = 0            # taken, not yet released

    @property
    def full(self):
        return self.captured + self.taken == self.slots

    def capture(self, tensor):
        """Enqueue the pack of `tensor` ([1][1][nz][ny][nx] CUDA float32) on the current stream and its copy to the
        next free slot; returns the frame's index.  Never waits."""
        c = tfluids._ctx_for(tensor)
        if c is not self.ctx:
            raise TflError("FrameRecorder: the tensor lives on another device than the recorder")
        assert tensor.dim() == 5 and tensor.is_contiguous(), "FrameRecorder: a contiguous 5-D tensor is needed"
        idx = C.c_int64(-1)
        self.ctx.check(self.ctx.lib.tfl_recorder_capture(self.ctx.h, self.h, tfluids._grid(tensor), C.byref(idx)))
        self.captured += 1
        return idx.value

    def take(self, wait=True):
        """-> (index, frame) of the oldest captured frame, or None if wait is false and its copy has not landed.
        frame is a [nx][ny][nz] numpy VIEW of pinned memory (`.vbox` order, `a[0, 0].transpose(2, 1, 0)` of the
        grid), valid until `release`: copy it to keep it."""
        ptr = C.POINTER(C.c_float)()
        idx = C.c_int64(-1)
        rc = self.ctx.lib.tfl_recorder_take(self.ctx.h, self.h, 1 if wait else 0, C.byref(ptr), C.byref(idx))
        if rc != 0 and idx.value >= 0:       # a z-slab frame whose planes did not all arrive: taken, to be released
            self.captured -= 1
            self.taken += 1
        self.ctx.check(rc)
        if idx.value < 0:
            return None
        self.captured -= 1
        self.taken += 1
        nz, ny, nx = self.shape
        return idx.value, np.ctypeslib.as_array(ptr, shape=(nx, ny, nz))

    def release(self):
        """Give back the slot of the oldest taken frame (its view must not be used afterwards)."""
        self.ctx.check(self.ctx.lib.tfl_recorder_release(self.ctx.h, self.h))
        self.taken -= 1

    def drain(self, writer, wait=False):
        """Write every captured frame whose copy has landed to `writer` (a formats.VboxWriter) in capture order;
        with wait, all of them.  Returns the number written."""
        n = 0
        while self.captured:
            got = self.take(wait)
            if got is None:
                break
            writer.write_packed(got[1])
            self.release()
            n += 1
        return n

    def record(self, tensor, writer):
        """capture, after writing the oldest frame to `writer` (waiting for its copy) if every slot is in use."""
        if self.full and self.captured:
            idx, frame = self.take(True)
            writer.write_packed(frame)
            self.release()
        return self.capture(tensor)

    def close(self):
        """Wait for the copies in flight and free the recorder (frames not taken are dropped)."""
        if getattr(self, "h", None):
            self.ctx.lib.tfl_recorder_destroy(self.ctx.h, self.h)
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


class SlabFrameRecorder(FrameRecorder):
    """One `.vbox` frame gathered from every rank of a z-slab run (tfl_recorder_create_slab, DESIGN.md section 6a).

    Every rank packs the global planes it owns (SlabDecomposition's z0 .. z1) straight into rank 0's staging frame;
    rank 0 is the writer and alone takes, releases, drains and records frames -- on the other ranks `record` is a
    capture and `drain` writes nothing.  Captures are collective: every rank captures the same number of times, in
    step order.  The constructor is collective too: rank 0's handle goes to the other ranks with `share` (by default
    torch.distributed over `group`) and it ends with `barrier`, so no rank captures before every rank is connected.
    `close` is collective as well: the other ranks free their recorders before rank 0 frees the frame they write into.

        rec = SlabFrameRecorder((gnz, ny, nx), rank, world)
        rec.record(local_density, z_offset, writer if rank == 0 else None)
    """

    def __init__(self, shape, rank, world, slots=3, device=None, group=None, share=None, barrier=None):
        """shape: the GLOBAL (gnz, ny, nx).  share(handle bytes on rank 0, None elsewhere) -> rank 0's bytes on every
        rank and barrier() replace torch.distributed (e.g. processes that share one GPU without a process group).
        Raises TflError on every rank if any rank could not map rank 0's frame (there is no other transport)."""
        import torch.distributed as dist
        shape = tuple(int(v) for v in shape)
        if len(shape) != 3:
            raise TflError("SlabFrameRecorder: shape must be the global (gnz, ny, nx), got %r" % (shape,))
        self.shape, self.rank, self.world, self.slots = shape, int(rank), int(world), int(slots)
        self.group = group
        self.ctx = tfluids.context(device)
        self.captured = 0
        self.taken = 0
        h = C.c_void_p()
        self.ctx.check(self.ctx.lib.tfl_recorder_create_slab(self.ctx.h, shape[0], shape[1], shape[2], self.rank,
                                                             self.world, self.slots, C.byref(h)))
        self.h = h
        if self.world == 1:
            return
        if share is None:
            def share(b):
                obj = [b]
                dist.broadcast_object_list(obj, src=0, group=group)
                return obj[0]
        self._custom = barrier is not None
        self._barrier = barrier or (lambda: dist.barrier(group=group))
        lib, error = self.ctx.lib, None
        if self.rank == 0:
            buf = C.create_string_buffer(_lib.RECORDER_HANDLE_BYTES)
            if lib.tfl_recorder_ipc_export(self.ctx.h, self.h, buf) != 0:
                error = lib.tfl_last_error(self.ctx.h).decode()
            handle = share(None if error else buf.raw)
        else:
            handle = share(None)
            if handle is None:
                error = "rank 0 could not export its frame"
            elif lib.tfl_recorder_ipc_connect(self.ctx.h, self.h, handle) != 0:
                error = lib.tfl_last_error(self.ctx.h).decode()
        if self._custom:                      # the barrier before the first capture; each rank reports its own error
            self._barrier()
            failed = [(self.rank, error)] if error else []
        else:                                 # every rank learns every rank's error (also the barrier)
            errs = [None] * self.world
            dist.all_gather_object(errs, error, group=group)
            failed = [(r, e) for r, e in enumerate(errs) if e]
        if failed:                            # nothing was captured: no rank writes into rank 0's frame
            self.ctx.lib.tfl_recorder_destroy(self.ctx.h, self.h)
            self.h = None
            raise TflError("SlabFrameRecorder: peer memory refused (%s); frames cannot be gathered asynchronously"
                           % "; ".join("rank %d: %s" % rf for rf in failed))

    def capture(self, tensor, z_offset):
        """Enqueue the pack of this rank's planes of `tensor` (its local [1][1][nz][ny][nx] CUDA float32 slab, whose
        plane 0 is global plane z_offset) on the current stream; returns the frame's index.  Never waits on the
        host."""
        c = tfluids._ctx_for(tensor)
        if c is not self.ctx:
            raise TflError("SlabFrameRecorder: the tensor lives on another device than the recorder")
        assert tensor.dim() == 5 and tensor.is_contiguous(), "SlabFrameRecorder: a contiguous 5-D tensor is needed"
        self.ctx.use_current_stream()
        return self.capture_grid(tfluids._grid(tensor), z_offset)

    def capture_grid(self, grid, z_offset):
        """capture of a tfl_grid (e.g. a field of tfl_slab_sim_layout) on the context's stream."""
        idx = C.c_int64(-1)
        self.ctx.check(self.ctx.lib.tfl_recorder_capture_slab(self.ctx.h, self.h, C.byref(grid), int(z_offset),
                                                              C.byref(idx)))
        if self.rank == 0:
            self.captured += 1
        return idx.value

    def drain(self, writer, wait=False):
        return super().drain(writer, wait) if self.rank == 0 else 0

    def _make_room(self, writer):
        if self.rank == 0 and self.full and self.captured:
            idx, frame = self.take(True)
            writer.write_packed(frame)
            self.release()

    def record(self, tensor, z_offset, writer):
        """capture on every rank; on rank 0 first writes the oldest frame to `writer` if every slot is in use."""
        self._make_room(writer)
        return self.capture(tensor, z_offset)

    def record_grid(self, grid, z_offset, writer):
        self._make_room(writer)
        return self.capture_grid(grid, z_offset)

    def close(self):
        """Free the recorder.  Collective for world > 1: the other ranks drain their packs and unmap, then (after a
        barrier) rank 0 waits for its copies and frees the frame."""
        if not getattr(self, "h", None):
            return
        if self.world > 1 and self.rank > 0:
            self.ctx.lib.tfl_recorder_destroy(self.ctx.h, self.h)
            self.h = None
        if self.world > 1 and getattr(self, "_barrier", None) is not None:
            self._barrier()
        if self.h:
            self.ctx.lib.tfl_recorder_destroy(self.ctx.h, self.h)
            self.h = None

    def __del__(self):
        pass          # close() is collective: never from the garbage collector
