"""On-disk formats on either side of the simulation loop (SURVEY.md section 8f-3), host side only.

* Manta frame dumps `*.bin` read by torch.loadMantaFile (torch/lib/load_manta_file.lua:15-60): five int32
  (transpose [legacy], nx, ny, nz, is3D), then Ux, Uy, [Uz], p as float32, flags as int32, density as
  float32, each nx*ny*nz values with x fastest.  The reference's dataset and its test data
  (tfluids/test_tfluids.lua: loadMantaBatch) use this layout.
* `.vbox` volumes written by the 3-D demo (torch/fluid_net_3d_sim.lua:155-172, 283-290): four int32
  (res x, res y, res z, number of frames) followed per frame by res^3 float32 permuted to x-SLOWEST order
  (`permute(3, 2, 1)` of the [z][y][x] grid).
"""
import struct

import numpy as np


def load_manta_file(path):
    """-> (p, U, flags, density, is3D) as float32 arrays shaped [1][c][nz][ny][nx] like torch.loadMantaFile
    (flags converted from int32 to float bit codes, U = cat(Ux, Uy[, Uz]) on the channel axis)."""
    with open(path, "rb") as f:
        head = f.read(20)
        if len(head) != 20:
            raise ValueError("%s: truncated header" % path)
        _transpose, nx, ny, nz, is3d = struct.unpack("<5i", head)
        numel = nx * ny * nz
        if min(nx, ny, nz) < 1 or is3d not in (0, 1):
            raise ValueError("%s: bad header %r" % (path, (nx, ny, nz, is3d)))

        def rd(dtype):
            a = np.fromfile(f, dtype=dtype, count=numel)
            if a.size != numel:
                raise ValueError("%s: truncated field" % path)
            return a.reshape(1, 1, nz, ny, nx)

        comps = [rd(np.float32), rd(np.float32)]
        if is3d:
            comps.append(rd(np.float32))
        p = rd(np.float32)
        flags = rd(np.int32).astype(np.float32)
        density = rd(np.float32)
    U = np.ascontiguousarray(np.concatenate(comps, axis=1))
    return p, U, flags, density, bool(is3d)


def save_manta_file(path, p, U, flags, density):
    """Inverse of load_manta_file (single batch element)."""
    nz, ny, nx = p.shape[-3:]
    is3d = U.shape[1] == 3
    with open(path, "wb") as f:
        f.write(struct.pack("<5i", 0, nx, ny, nz, 1 if is3d else 0))
        for c in range(U.shape[1]):
            np.ascontiguousarray(U[0, c], np.float32).tofile(f)
        np.ascontiguousarray(p[0, 0], np.float32).tofile(f)
        np.ascontiguousarray(flags[0, 0]).astype(np.int32).tofile(f)
        np.ascontiguousarray(density[0, 0], np.float32).tofile(f)


class VboxWriter:
    """Streaming `.vbox` writer: header first, then one frame per `write` ([z][y][x] or [1][c][z][y][x],
    multi-channel density averaged over the channels as the demo does)."""

    def __init__(self, path, res, num_frames):
        rx, ry, rz = (res, res, res) if np.isscalar(res) else res
        self.shape = (rz, ry, rx)
        self.f = open(path, "wb")
        self.f.write(struct.pack("<4i", rx, ry, rz, num_frames))

    def write(self, frame):
        a = np.asarray(frame, np.float32)
        if a.ndim == 5:
            a = a[0].mean(axis=0)
        assert a.shape == self.shape, (a.shape, self.shape)
        np.ascontiguousarray(a.transpose(2, 1, 0)).tofile(self.f)      # permute(3, 2, 1): x slowest

    def write_packed(self, frame):
        """One frame already in file order, [x][y][z] (a record.FrameRecorder frame)."""
        a = np.asarray(frame)
        assert a.dtype == np.float32 and a.shape == self.shape[::-1], (a.dtype, a.shape, self.shape[::-1])
        np.ascontiguousarray(a).tofile(self.f)

    def close(self):
        self.f.close()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


def load_vbox(path):
    """-> array [frames][z][y][x] (undoing the x-slowest permutation)."""
    with open(path, "rb") as f:
        rx, ry, rz, frames = struct.unpack("<4i", f.read(16))
        a = np.fromfile(f, dtype=np.float32)
    n = a.size // (rx * ry * rz)
    return a[:n * rx * ry * rz].reshape(n, rx, ry, rz).transpose(0, 3, 2, 1)


def load_binvox(path):
    """tfluids.loadVoxelData (torch/lib/obstacles_import_binvox.lua:39-120): a `.binvox` occupancy volume
    (ASCII header `#binvox 1` / `dim a b c` / `translate ...` / `scale s` / `data`, then run-length pairs
    (value byte, count byte)) -> {'dims', 'translation', 'scale', 'data'} with data float32 of shape
    [dims0][dims2][dims1] (the reference's `view(d0, d1, d2):permute(1, 3, 2)`).

    Restated with the reference parser's behaviour, not the format's ideal: a run writes its value to
    `count + 1` cells (the extra cell is overwritten by the next run) and the LAST run of the file is
    dropped, because the loop stops writing once the read position reaches the end of the file
    (`if (file:position() < endPosition)`, :93) -- so the cell after the second-to-last run keeps that
    run's value and the rest of the last run stays 0.  Kept for byte-exact reproduction of what the
    reference feeds its simulations."""
    with open(path, "rb") as f:
        raw = f.read()
    pos = 0
    lines = []
    for _ in range(5):
        end = raw.index(b"\n", pos)
        lines.append(raw[pos:end].decode("ascii").strip())
        pos = end + 1
    if not lines[0].startswith("#binvox"):
        raise ValueError("%s: not a binvox file" % path)
    dims = [int(v) for v in lines[1].split()[1:4]]
    translation = [float(v) for v in lines[2].split()[1:4]]
    scale = float(lines[3].split()[1])
    count_total = dims[0] * dims[1] * dims[2]
    data = np.zeros(count_total + 1, np.uint8)
    body = raw[pos:]
    index = 0                     # 0-based version of the reference's 1-based `index`
    end_index = 0
    read = 0
    while end_index + 1 < count_total and read + 2 <= len(body):
        value, count = body[read], body[read + 1]
        read += 2
        if read < len(body):      # the reference's position test: the final pair is read but not applied
            end_index = index + count
            if end_index + 1 > count_total:
                raise ValueError("%s: run-length data overruns the volume" % path)
            data[index:end_index + 1] = value
            index = end_index
    vol = data[:count_total].reshape(dims[0], dims[1], dims[2]).transpose(0, 2, 1)
    return {"dims": dims, "translation": translation, "scale": scale,
            "data": np.ascontiguousarray(vol, np.float32)}


# ---- placing a voxelised obstacle in a domain (torch/lib/voxel_utils.lua), restated literally: the demo's scenes
# (torch/fluid_net_3d_sim.lua:92-132) are built with these.  Volumes are 3-D arrays indexed [d1][d2][d3] like the
# Torch tensors (Lua's dims 1, 2, 3); the demo's padded volume is [z][y][x] of the grid.

def calculate_bounding_box(voxels):
    """tfluids.calculateBoundingBox (voxel_utils.lua:20-50): {'min': [m1, m2, m3], 'max': [M1, M2, M3]}, per axis the
    first and last 1-based index whose slab (the sum over the other two axes) is non-zero.  An empty volume fails the
    reference's assertion."""
    v = np.asarray(voxels)
    assert v.ndim == 3

    def first_last_nonzero(data):
        nz = np.flatnonzero(data != 0)
        return (int(nz[0]) + 1, int(nz[-1]) + 1) if nz.size else (None, None)

    # the reference's xmin / ymin / zmin are Lua dims 1 / 2 / 3 (voxels:sum(2):sum(3), :sum(1):sum(3), :sum(1):sum(2))
    s = v.astype(np.float64)
    mins, maxs = [], []
    for axis in range(3):
        lo, hi = first_last_nonzero(s.sum(axis=tuple(a for a in range(3) if a != axis)))
        mins.append(lo)
        maxs.append(hi)
    assert s.sum() > 0                       # make sure the volume wasn't empty
    return {"min": mins, "max": maxs}


def pad_voxels_to_dims(width, height, depth, voxels, offsetX, offsetY, offsetZ):
    """tfluids.padVoxelsToDims (voxel_utils.lua:176-203): the volume trimmed to its bounding box and pasted into a
    zeroed [depth][height][width] grid, before-padding max(floor((extent - size) / 2 + offset), 1) per axis (x: width,
    Lua dim 3; y: height, dim 2; z: depth, dim 1).  Offsets may be negative or fractional; the clamp keeps at least one
    empty plane before the volume.  A paste that would reach past the grid fails (the reference's tensor indexing
    does); the reference's closing check that no voxel was lost is kept."""
    v = np.asarray(voxels)
    assert v.ndim == 3
    assert v.shape[0] <= depth and v.shape[1] <= height and v.shape[2] <= width
    bbox = calculate_bounding_box(v)
    (a1, a2, a3), (b1, b2, b3) = bbox["min"], bbox["max"]
    v = np.ascontiguousarray(v[a1 - 1:b1, a2 - 1:b2, a3 - 1:b3])
    pad_lft = max(int(np.floor((width - v.shape[2]) / 2 + offsetX)), 1)
    pad_bot = max(int(np.floor((height - v.shape[1]) / 2 + offsetY)), 1)
    pad_bck = max(int(np.floor((depth - v.shape[0]) / 2 + offsetZ)), 1)
    for pad, size, extent, name in ((pad_bck, v.shape[0], depth, "depth"), (pad_bot, v.shape[1], height, "height"),
                                    (pad_lft, v.shape[2], width, "width")):
        if pad + size > extent:
            raise IndexError("padVoxelsToDims: the volume (%d cells after %d of padding) does not fit the %s %d"
                             % (size, pad, name, extent))
    ret = np.zeros((depth, height, width), v.dtype)
    ret[pad_bck:pad_bck + v.shape[0], pad_bot:pad_bot + v.shape[1], pad_lft:pad_lft + v.shape[2]] = v
    assert ret.sum(dtype=np.float64) == v.sum(dtype=np.float64), "Lost some voxels."
    return ret


def flip_diagonal(voxels, axis):
    """tfluids.flipDiagonal (voxel_utils.lua:225-277), in place: axis 0 swaps Lua dims 2 and 3 (needs them equal),
    axis 1 dims 1 and 3, axis 2 dims 1 and 2.  Returns `voxels`."""
    dims = voxels.shape
    assert len(dims) == 3
    assert 0 <= axis <= 2
    if axis == 0:
        assert dims[1] == dims[2]
    elif axis == 1:
        assert dims[0] == dims[2]
    else:
        assert dims[0] == dims[1]
    perm = {0: (0, 2, 1), 1: (2, 1, 0), 2: (1, 0, 2)}[axis]
    voxels[...] = np.ascontiguousarray(voxels.transpose(perm))
    return voxels
