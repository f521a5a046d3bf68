"""Density frames of z-slab runs (tfl_recorder_create_slab / _capture_slab, record.SlabFrameRecorder, the scene's slab
mode) on the GPU: the cross-rank protocol with several processes sharing cuda:0, the refusals, the world-1 slab scene
against the single-GPU scene, convnet frames against synchronous downloads, and 2- / 4-GPU runs where the box has the
GPUs."""
import ctypes as C
import os
import socket
import time

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from fluidnet_b200 import record, scene, synth, tfluids
from fluidnet_b200._lib import TflError

pytestmark = pytest.mark.gpu

GHOST = 0x7FBADBAD          # a NaN payload that fills ghost planes and must never reach a frame
AFTER = 0x7F80DEAD          # written over the field right after each capture


def special_bits(shape, seed):
    """Random float32 bit patterns with -0.0, denormals and NaN payloads at the front (as test_gpu_record.py)."""
    bits = np.random.default_rng(seed).integers(0, 2 ** 32, size=shape, dtype=np.uint64).astype(np.uint32)
    flat = bits.reshape(-1)
    specials = np.array([0x80000000, 0x00000001, 0x007FFFFF, 0x80000001, 0x7FC12345, 0x7F800001, 0xFFBADBAD], np.uint32)
    flat[:min(flat.size, specials.size)] = specials[:flat.size]
    return bits


def _collect(procs, q, timeout_s):
    """Results of all ranks; if one rank fails (or time runs out) the others are killed (test_gpu_slab.py's pattern)."""
    import queue
    res, t0 = [], time.time()
    while len(res) < len(procs) and time.time() - t0 < timeout_s:
        try:
            r = q.get(timeout=1.0)
            res.append(r)
            if r[1] != "ok":
                break
        except queue.Empty:
            if any(p.exitcode not in (None, 0) for p in procs):
                break
    for p in procs:
        p.join(5 if len(res) == len(procs) else 0.1)
        if p.is_alive():
            p.kill()
    return res


def _protocol_worker(rank, world, shape, frames, q, qh, barrier, slow_rank):
    """One rank of a z-slab recorder on cuda:0.  Its local slab comes from SlabDecomposition (owned planes of the
    frame's global field, ghost planes of GHOST bits); rank 0 checks every frame against the global field."""
    try:
        from fluidnet_b200.slab import SlabDecomposition
        torch.cuda.set_device(0)
        gnz, ny, nx = shape
        dec = SlabDecomposition(gnz, rank, world, halo=2)

        def share(b):
            if rank == 0:
                for _ in range(world - 1):
                    qh.put(b)
                return b
            return qh.get(timeout=120)

        checked = 0
        stream = torch.cuda.Stream()
        with torch.cuda.stream(stream):
            local = torch.empty(1, 1, dec.nz, ny, nx, device="cuda")
            for slots in (1, 2, 3):
                rec = record.SlabFrameRecorder(shape, rank, world, slots, share=share, barrier=barrier.wait)
                got = {}

                def take_one():
                    idx, frame = rec.take(wait=True)
                    got[idx] = frame.view(np.uint32).copy()
                    rec.release()

                for f in range(frames):
                    glob = special_bits(shape, 1000 * slots + f)
                    arr = np.full((dec.nz, ny, nx), GHOST, np.uint32)
                    arr[dec.own_lo:dec.own_hi] = glob[dec.z0:dec.z1]
                    local.copy_(torch.from_numpy(arr.view(np.float32)).view(1, 1, dec.nz, ny, nx))
                    if rank == 0 and rec.full:
                        take_one()
                    barrier.wait()                       # every rank starts the round together ...
                    if rank == slow_rank:
                        time.sleep(0.03)                 # ... but one of them packs a few tens of ms late
                    assert rec.capture(local, dec.zoff) == f
                    local.view(torch.int32).fill_(AFTER)
                if rank == 0:
                    while rec.captured:
                        take_one()
                    assert sorted(got) == list(range(frames))
                    for f in range(frames):
                        want = special_bits(shape, 1000 * slots + f).transpose(2, 1, 0)
                        assert got[f].shape == want.shape and np.array_equal(got[f], want), (slots, f)
                        checked += 1
                stream.synchronize()
                rec.close()                              # collective: the other ranks unmap before rank 0 frees
            assert tfluids.context().trace_faults() == 0
        q.put((rank, "ok", checked))
    except Exception:               # pragma: no cover
        import traceback
        q.put((rank, "FAIL: %s" % traceback.format_exc(), 0))
        raise


@pytest.mark.parametrize("world,shape", [(2, (33, 5, 7)), (3, (70, 9, 31)), (5, (97, 65, 129))])
def test_slab_frames_from_several_processes_on_one_gpu(world, shape):
    """Processes sharing cuda:0, each with its own context, gather 12 frames per ring size (1, 2, 3 slots) into rank
    0's recorder; every frame equals its global field in `.vbox` order bit for bit.  Without MPS the processes
    time-slice the GPU, so frames are small and a barrier starts each round: every wait ends far inside its bound."""
    ctx = mp.get_context("spawn")
    q, qh, barrier = ctx.Queue(), ctx.Queue(), ctx.Barrier(world)
    procs = [ctx.Process(target=_protocol_worker, args=(r, world, shape, 12, q, qh, barrier, world - 1))
             for r in range(world)]
    for p in procs:
        p.start()
    res = _collect(procs, q, 300)
    assert len(res) == world and all(r[1] == "ok" for r in res), res
    assert sum(r[2] for r in res) == 36


def _create_slab(ctx, gnz, ny, nx, rank, world, slots):
    h = C.c_void_p()
    rc = ctx.lib.tfl_recorder_create_slab(ctx.h, gnz, ny, nx, rank, world, slots, C.byref(h))
    return rc, h


def test_refusals_launch_nothing():
    ctx = tfluids.context()
    lib = ctx.lib
    msg = lambda: lib.tfl_last_error(ctx.h).decode()       # noqa: E731
    rc, h = _create_slab(ctx, 3, 4, 4, 0, 4, 2)
    assert rc != 0 and h.value is None and "empty slabs" in msg()
    rc, h = _create_slab(ctx, 130, 4, 4, 0, 65, 2)
    assert rc != 0 and h.value is None and "world 65" in msg()
    rc, h = _create_slab(ctx, 16, 4, 4, 0, 2, 0)
    assert rc != 0 and h.value is None and "slots" in msg()

    d = torch.zeros(1, 1, 16, 4, 4, device="cuda")
    l0 = ctx.launch_count()
    # rank 1 of 2, not connected; take / release / export refused by name
    rc, r1 = _create_slab(ctx, 16, 4, 4, 1, 2, 0)
    assert rc == 0
    idx = C.c_int64(7)
    assert lib.tfl_recorder_capture_slab(ctx.h, r1, C.byref(tfluids._grid(d)), 0, C.byref(idx)) != 0
    assert "not connected" in msg() and idx.value == -1
    ptr = C.POINTER(C.c_float)()
    assert lib.tfl_recorder_take(ctx.h, r1, 1, C.byref(ptr), C.byref(idx)) != 0 and "rank 0 (the writer) takes" in msg()
    assert lib.tfl_recorder_release(ctx.h, r1) != 0 and "rank 0 (the writer) releases" in msg()
    buf = C.create_string_buffer(128)
    assert lib.tfl_recorder_ipc_export(ctx.h, r1, buf) != 0 and "rank 1 does not export" in msg()
    # rank 0 of 2 before export; the whole-grid capture refuses a z-slab recorder
    rc, r0 = _create_slab(ctx, 16, 4, 4, 0, 2, 2)
    assert rc == 0
    assert lib.tfl_recorder_capture_slab(ctx.h, r0, C.byref(tfluids._grid(d)), 0, C.byref(idx)) != 0
    assert "not connected" in msg()
    assert lib.tfl_recorder_capture(ctx.h, r0, C.byref(tfluids._grid(d)), C.byref(idx)) != 0
    assert "tfl_recorder_capture_slab" in msg()
    assert lib.tfl_recorder_ipc_connect(ctx.h, r0, buf) != 0 and "rank 0 (the writer) exports" in msg()
    assert lib.tfl_recorder_ipc_export(ctx.h, r0, buf) == 0
    # a handle of another shape or world is refused by name before anything is mapped
    for gnz, world, rank in ((17, 2, 1), (16, 3, 1)):
        rc, other = _create_slab(ctx, gnz, 4, 4, rank, world, 0)
        assert rc == 0
        assert lib.tfl_recorder_ipc_connect(ctx.h, other, buf) != 0
        assert "handle is of a 16 x 4 x 4 recorder over 2 ranks" in msg(), msg()
        lib.tfl_recorder_destroy(ctx.h, other)
    assert lib.tfl_recorder_ipc_connect(ctx.h, r1, b"\0" * 128) != 0 and "not a recorder's handle" in msg()
    lib.tfl_recorder_destroy(ctx.h, r1)
    lib.tfl_recorder_destroy(ctx.h, r0)
    assert ctx.launch_count() == l0

    # world 1 (rank 0 owns [0, 16)): field refusals, graph capture, full ring and its retry
    rec = record.SlabFrameRecorder((16, 4, 4), 0, 1, slots=1)
    l0 = ctx.launch_count()
    with pytest.raises(TflError, match=r"from global plane 1 does not hold rank 0's planes \[0, 16\)"):
        rec.capture(torch.zeros(1, 1, 16, 4, 4, device="cuda"), 1)
    with pytest.raises(TflError, match="a field of 15 planes"):
        rec.capture(torch.zeros(1, 1, 15, 4, 4, device="cuda"), 0)
    with pytest.raises(TflError, match=r"field planes are 4 x 5 \(y, x\)"):
        rec.capture(torch.zeros(1, 1, 16, 4, 5, device="cuda"), 0)
    with pytest.raises(TflError, match="nb = 2"):
        rec.capture(torch.zeros(2, 1, 16, 4, 4, device="cuda"), 0)
    with pytest.raises(TflError, match="nc = 3"):
        rec.capture(torch.zeros(1, 3, 16, 4, 4, device="cuda"), 0)
    side = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        ctx.use_current_stream()               # the context adopts the stream before its capture begins
        with pytest.raises(TflError, match="captured into a graph"):
            with torch.cuda.graph(g, stream=side):
                rec.capture(d, 0)
    assert ctx.launch_count() == l0
    d.copy_(torch.arange(256, dtype=torch.float32, device="cuda").view(1, 1, 16, 4, 4))
    ctx.use_current_stream()
    assert rec.capture(d, 0) == 0
    l1 = ctx.launch_count()
    with pytest.raises(TflError, match=r"recorder's 1 slot\(s\)"):
        rec.capture(d, 0)
    assert ctx.launch_count() == l1
    idx0, frame = rec.take(wait=True)
    assert idx0 == 0 and np.array_equal(frame, d.cpu().numpy()[0, 0].transpose(2, 1, 0))
    rec.release()
    assert rec.capture(d, 0) == 1                           # the refused capture did not use up a frame number
    idx1, _ = rec.take(wait=True)
    assert idx1 == 1
    rec.release()
    rec.close()


def _scene_files(out):
    blobs = {}
    for k in ("density", "geom", "geom_blender"):
        with open(out[k], "rb") as f:
            blobs[k] = f.read()
    return blobs


@pytest.mark.parametrize("res", [32, 48])
def test_world1_slab_scene_equals_the_single_gpu_scene(res, tmp_path):
    """The jacobi scene on one z-slab rank (tfl_slab_sim_step, bit-identical to tfl_simulate_step) writes the
    single-GPU scene's files byte for byte."""
    frames = 30
    one = scene.run(res, "plume", "jacobi", None, None, "none", str(tmp_path / "one"), None, frames, 3,
                    log=lambda *a: None)
    slab = scene.run(res, "plume", "jacobi", None, None, "none", str(tmp_path / "slab"), None, frames, 3,
                     log=lambda *a: None, slabs=True, world=1, rank=0)
    assert slab["frames_written"] == one["frames_written"] == 10
    assert os.path.basename(slab["density"]) == os.path.basename(one["density"])
    a, b = _scene_files(one), _scene_files(slab)
    for k in a:
        assert a[k] == b[k], k
    assert len(a["density"]) == 16 + 10 * res ** 3 * 4


def test_world1_convnet_frames_equal_synchronous_downloads():
    """Every frame recorded from a convnet slab run equals a synchronous download of the same run at the same step."""
    from fluidnet_b200.model import ProjectionModel
    from fluidnet_b200.slab import NativeSlabSimulator
    from fluidnet_b200 import simulate
    n = 32
    flags = scene.scene_flags(n)
    z = lambda c: torch.zeros(1, c, n, n, n)       # noqa: E731
    batch = {"pDiv": z(1), "UDiv": z(3), "flags": torch.from_numpy(flags), "density": z(1)}
    simulate.createPlumeBCs(batch, [1], n / 128, 0.15)
    model = ProjectionModel(synth.make_model(True)["layers"], True)
    mconf = scene.scene_mconf(n, "convnet")
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        sim = NativeSlabSimulator(batch, mconf, None, torch.device("cuda", 0), 0, 1, 3, model=model)
        rec = sim.frame_recorder(slots=2)
        want = {}
        for step in range(12):
            sim.step()
            for key in ("density", "pDiv"):
                if rec.full:
                    idx, frame = rec.take(wait=True)
                    assert np.array_equal(frame.view(np.uint32), want.pop(idx)), idx
                    rec.release()
                idx = sim.record(rec, None, key)
                want[idx] = sim.gather(key).numpy()[0, 0].transpose(2, 1, 0).view(np.uint32).copy()
        while rec.captured:
            idx, frame = rec.take(wait=True)
            assert np.array_equal(frame.view(np.uint32), want.pop(idx)), idx
            rec.release()
        assert not want
        assert sim.gather("density").abs().max().item() > 0
        sim.check()
        rec.close()
        sim.close()


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _gpu_worker(rank, world, port, out_dir, q):
    try:
        import torch.distributed as dist
        from fluidnet_b200.model import ProjectionModel
        from fluidnet_b200.slab import NativeSlabSimulator
        from fluidnet_b200 import simulate
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        torch.cuda.set_device(rank)
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
        res = 64
        slab = scene.run(res, "plume", "jacobi", None, None, "none", os.path.join(out_dir, "slab"), None, 18, 3,
                         log=lambda *a: None, slabs=True, world=world, rank=rank)
        flags = scene.scene_flags(res)
        z = lambda c: torch.zeros(1, c, res, res, res)       # noqa: E731
        batch = {"pDiv": z(1), "UDiv": z(3), "flags": torch.from_numpy(flags), "density": z(1)}
        simulate.createPlumeBCs(batch, [1], res / 128, 0.15)
        model = ProjectionModel(synth.make_model(True)["layers"], True)
        stream = torch.cuda.Stream()
        mism = 0
        with torch.cuda.stream(stream):
            sim = NativeSlabSimulator(batch, scene.scene_mconf(res, "convnet"), None, torch.device("cuda", rank), rank,
                                      world, 3, model=model)
            assert sim.halo_transport.startswith("peer memory"), sim.halo_transport
            rec = sim.frame_recorder(slots=2)
            want = {}
            for step in range(8):
                sim.step()
                idx = sim.record(rec, None)
                g = sim.gather("density")
                if rank == 0:
                    want[idx] = g.numpy()[0, 0].transpose(2, 1, 0).view(np.uint32).copy()
                    idx, frame = rec.take(wait=True)
                    mism += not np.array_equal(frame.view(np.uint32), want.pop(idx))
                    rec.release()
            sim.check()
            rec.close()
            sim.close()
        if rank == 0:
            one = scene.run(res, "plume", "jacobi", None, None, "none", os.path.join(out_dir, "one"), None, 18, 3,
                            log=lambda *a: None, world=1, rank=0)
            a, b = _scene_files(one), _scene_files(slab)
            assert all(a[k] == b[k] for k in a), [k for k in a if a[k] != b[k]]
            assert mism == 0, mism
        dist.barrier()
        dist.destroy_process_group()
        q.put((rank, "ok"))
    except Exception:               # pragma: no cover
        import traceback
        q.put((rank, "FAIL: %s" % traceback.format_exc()))
        raise


@pytest.mark.parametrize("world", [2, 4])
def test_multi_gpu_scene_and_frames(world, tmp_path):
    """world GPUs over peer memory: the jacobi scene's files equal the single-GPU scene's byte for byte, and convnet
    frames equal gather('density') of the same run."""
    if torch.cuda.device_count() < world:
        pytest.skip("needs %d GPUs" % world)
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_gpu_worker, args=(r, world, port, str(tmp_path), q)) for r in range(world)]
    for p in procs:
        p.start()
    res = _collect(procs, q, 300)
    assert len(res) == world and all(r[1] == "ok" for r in res), res
