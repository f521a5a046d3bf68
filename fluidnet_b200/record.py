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

from . import tfluids
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
        self.ctx.check(self.ctx.lib.tfl_recorder_take(self.ctx.h, self.h, 1 if wait else 0, C.byref(ptr), C.byref(idx)))
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
