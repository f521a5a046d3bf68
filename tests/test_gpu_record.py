"""The frame recorder (tfl_recorder_*, fluidnet_b200/record.py) and the demo scene (fluidnet_b200/scene.py) on the GPU:
k_pack_vbox as a bit copy into `.vbox` order, stream order behind replayed step graphs, no host or device waits the
caller did not ask for, refusals that launch nothing, the recorder's lifecycle, and the scene's files against a plain
synchronous loop."""
import time

import numpy as np
import pytest
import torch

from fluidnet_b200 import formats, record, scene, simulate, synth, tfluids
from fluidnet_b200._lib import TflError
from fluidnet_b200.model import ProjectionModel

pytestmark = pytest.mark.gpu


def special_bits(shape, seed):
    """float32 values as raw bits: random words (NaNs with payloads, denormals, infinities included) and, at the
    front, -0.0, the smallest and largest denormals, a quiet and a signalling NaN with payloads."""
    bits = np.random.default_rng(seed).integers(0, 2 ** 32, size=shape, dtype=np.uint64).astype(np.uint32)
    flat = bits.reshape(-1)
    specials = np.array([0x80000000, 0x00000001, 0x007FFFFF, 0x80000001, 0x7FC12345, 0x7F800001, 0xFFBADBAD,
                         0x7F800000], np.uint32)
    flat[:min(flat.size, specials.size)] = specials[:flat.size]
    return bits


@pytest.mark.parametrize("nz,ny,nx", [(1, 1, 1), (1, 5, 7), (7, 9, 31), (33, 65, 129), (128, 128, 128)])
def test_pack_is_a_bit_copy_in_vbox_order(nz, ny, nx):
    bits = special_bits((1, 1, nz, ny, nx), nz * 131 + nx)
    a = torch.from_numpy(bits.view(np.float32)).cuda()
    ctx = tfluids.context()
    with record.FrameRecorder((nz, ny, nx), slots=2) as rec:
        l0 = ctx.launch_count()
        assert rec.capture(a) == 0
        assert ctx.launch_count() == l0 + 1
        idx, frame = rec.take(wait=True)
        assert idx == 0 and frame.shape == (nx, ny, nz)
        want = bits[0, 0].transpose(2, 1, 0)
        assert np.array_equal(frame.view(np.uint32), want)
        rec.release()


def plume_problem(n, seed=7):
    flags = synth.make_flags(n, n, n, True, nb=1, geometry=True, seed=seed)
    batch = {"pDiv": np.zeros_like(flags), "UDiv": synth.make_smooth_velocity(flags, True, amp=2.0), "flags": flags,
             "density": synth.make_density(flags)}
    gb = {k: torch.from_numpy(v.copy()).cuda() for k, v in batch.items()}
    simulate.createPlumeBCs(gb, [1.0], n / 128.0, 0.15)
    mconf = scene.scene_mconf(n)
    return gb, mconf


@pytest.fixture(scope="module")
def net():
    return ProjectionModel(synth.make_model(True)["layers"], True)


@pytest.mark.parametrize("slots", [1, 2, 3])
def test_frames_follow_stream_order_behind_replayed_steps(slots, net):
    """12 step-graph replays at 64^3, a capture after each, a stream-ordered device clone right after the capture;
    frames are taken only when the ring is full (lagging slots - 1 frames behind) and must equal their clones."""
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        gb, mconf = plume_problem(64)
        simulate.simulate_fused(None, mconf, gb, net)
        graph = simulate.StepGraph(mconf, gb, net)
        clones, got = [], {}
        with record.FrameRecorder(gb["density"].shape, slots=slots) as rec:
            for i in range(12):
                graph.launch()
                if rec.full:
                    idx, frame = rec.take(wait=True)
                    got[idx] = np.array(frame)
                    rec.release()
                assert rec.capture(gb["density"]) == i
                clones.append(gb["density"].clone())
            while rec.captured:
                idx, frame = rec.take(wait=True)
                got[idx] = np.array(frame)
                rec.release()
        graph.close()
        stream.synchronize()
    assert sorted(got) == list(range(12))
    for i, c in enumerate(clones):
        assert np.array_equal(got[i].view(np.uint32), c.cpu().numpy()[0, 0].transpose(2, 1, 0).view(np.uint32)), i
    assert not np.array_equal(got[0], got[11])         # the density moved between the first and the last frame


def test_capture_and_take_do_not_wait_for_the_device():
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        d = torch.rand(1, 1, 64, 64, 64, device="cuda")
        rec = record.FrameRecorder(d.shape, slots=2)
        a = torch.randn(4096, 4096, device="cuda")
        b = torch.randn(4096, 4096, device="cuda") / 64.0
        with record.FrameRecorder(d.shape, slots=1) as warm:     # the pack kernel and the matmul loaded beforehand
            warm.capture(d)
            warm.take(wait=True)
        a = a @ b
        stream.synchronize()
        for _ in range(20):                            # ~50 ms of ordinary matmuls queued ahead of the capture
            a = a @ b
        t0 = time.perf_counter()
        assert rec.capture(d) == 0
        returned = time.perf_counter() - t0
        assert not stream.query(), "the queued work finished before the capture returned: nothing was measured"
        assert rec.take(wait=False) is None
        assert not stream.query()
        stream.synchronize()
        got = rec.take(wait=False)
        assert got is not None and got[0] == 0
        assert np.array_equal(got[1], d.cpu().numpy()[0, 0].transpose(2, 1, 0))
        rec.release()
        rec.close()
    assert returned < 0.02, returned


def test_refusals_launch_nothing():
    ctx = tfluids.context()
    d = torch.zeros(1, 1, 8, 8, 8, device="cuda")
    with record.FrameRecorder((8, 8, 8), slots=1) as rec:
        l0 = ctx.launch_count()
        with pytest.raises(TflError, match="no taken frame"):
            rec.release()
        t0 = time.perf_counter()
        with pytest.raises(TflError, match="no captured frame"):
            rec.take(wait=True)
        assert time.perf_counter() - t0 < 1.0
        with pytest.raises(TflError, match="nb = 2"):
            rec.capture(torch.zeros(2, 1, 8, 8, 8, device="cuda"))
        with pytest.raises(TflError, match="nc = 3"):
            rec.capture(torch.zeros(1, 3, 8, 8, 8, device="cuda"))
        with pytest.raises(TflError, match="8 x 8 x 8"):
            rec.capture(torch.zeros(1, 1, 8, 8, 9, device="cuda"))
        assert ctx.launch_count() == l0
        rec.capture(d)
        l1 = ctx.launch_count()
        with pytest.raises(TflError, match=r"recorder's 1 slot\(s\)"):
            rec.capture(d)
        idx, _ = rec.take(wait=True)
        with pytest.raises(TflError, match="slot"):        # taken but not released still holds the slot
            rec.capture(d)
        assert ctx.launch_count() == l1
        rec.release()
        assert rec.capture(d) == 1
    for bad in ((0, 8, 8, 1), (8, 8, 8, 0)):
        with pytest.raises(TflError):
            record.FrameRecorder(bad[:3], slots=bad[3])
    import ctypes as C
    h = C.c_void_p(0x1234)
    assert ctx.lib.tfl_recorder_create(ctx.h, 8, 8, 8, 0, C.byref(h)) != 0 and h.value is None


def test_destroy_with_copies_in_flight_and_recreate():
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        d = torch.rand(1, 1, 128, 128, 128, device="cuda")
        rec = record.FrameRecorder(d.shape, slots=3)
        for _ in range(3):
            rec.capture(d)
        rec.close()                                     # waits for its copies, then frees
        for k in range(5):
            with record.FrameRecorder(d.shape, slots=2) as rec:
                rec.capture(d)
                rec.capture(d)
                if k % 2:
                    rec.take(wait=True)
        with record.FrameRecorder(d.shape, slots=1) as rec:
            rec.capture(d)
            idx, frame = rec.take(wait=True)
            assert np.array_equal(frame, d.cpu().numpy()[0, 0].transpose(2, 1, 0))
            rec.release()
        stream.synchronize()


def test_file_written_through_the_recorder_reads_back(tmp_path):
    path = str(tmp_path / "frames.vbox")
    frames = [torch.rand(1, 1, 12, 10, 14, device="cuda") for _ in range(7)]
    with record.FrameRecorder((12, 10, 14), slots=2) as rec, formats.VboxWriter(path, (14, 10, 12), 7) as w:
        for f in frames:
            rec.record(f, w)
            rec.drain(w)
        rec.drain(w, wait=True)
    got = formats.load_vbox(path)
    assert np.array_equal(got, np.stack([f.cpu().numpy()[0, 0] for f in frames]))


def plain_loop(res, sim_method, model, voxels, frames, decimation, path):
    """The demo's loop as the reference runs it: step, then every `decimation` frames a synchronous download and a
    VboxWriter write.  Convnet: frame 1 through simulate_fused, later frames replayed from a step graph."""
    mconf = scene.scene_mconf(res, sim_method)
    if model is not None:
        mconf["normalizeInputThreshold"] = float(model.threshold)
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        z = lambda c: torch.zeros(1, c, res, res, res, device="cuda")      # noqa: E731
        batch = {"pDiv": z(1), "UDiv": z(3), "flags": torch.from_numpy(scene.scene_flags(res, voxels)).cuda(),
                 "density": z(1)}
        simulate.createPlumeBCs(batch, [1], res / 128, 0.15)
        graph = None
        with formats.VboxWriter(path, res, frames) as w:
            for i in range(1, frames + 1):
                if graph is not None:
                    graph.launch()
                else:
                    simulate.simulate_fused(None, mconf, batch, model)
                if i == 1 and sim_method == "convnet":
                    graph = simulate.StepGraph(mconf, batch, model)
                if i % decimation == 0:
                    w.write(batch["density"].cpu().numpy())
        if graph is not None:
            graph.close()
        stream.synchronize()


@pytest.mark.parametrize("which,sim_method", [("plume", "convnet"), ("arch", "convnet"), ("plume", "jacobi"),
                                              ("bunny", "pcg")])
def test_scene_files_equal_a_plain_loop(which, sim_method, net, tmp_path, orc):
    from test_scene import write_binvox
    res, frames = 32, 9
    binvox = None
    if which != "plume":
        d = scene.model_res(res)
        occ = np.zeros((d, d, d), np.uint8)
        occ[3:12, 2:9, 4:13] = 1
        occ[5:8, 2:5, 6:9] = 0                                  # an arch-like opening at the bottom
        binvox = str(tmp_path / scene.binvox_name(which, res))
        write_binvox(binvox, (d, d, d), occ.reshape(-1))
    model = net if sim_method == "convnet" else None
    out = scene.run(res, which, sim_method, model, None, "synthetic", str(tmp_path / "out"), binvox, frames, 3,
                    log=lambda *a: None)
    assert out["density"].endswith("density_output_synthetic_dt0.1.vbox") and out["frames_written"] == 3
    want = str(tmp_path / "plain.vbox")
    voxels = scene.obstacle_voxels(which, res, binvox)
    if voxels is not None:
        assert voxels.sum() > 0
    plain_loop(res, sim_method, model, voxels, frames, 3, want)
    with open(out["density"], "rb") as f, open(want, "rb") as g:
        a, b = f.read(), g.read()
    assert a[:16] == b[:16] and np.frombuffer(a[:16], np.int32).tolist() == [res, res, res, frames]
    assert len(a) == 16 + 3 * res ** 3 * 4 and a == b
    dens = formats.load_vbox(out["density"])
    assert dens.shape[0] == 3 and dens[-1].max() > 0
    occ = orc.flagsToOccupancy(scene.scene_flags(res, voxels))[0, 0]
    geom, blender = formats.load_vbox(out["geom"]), formats.load_vbox(out["geom_blender"])
    assert geom.shape == (1, res, res, res) and np.array_equal(geom[0], occ)
    edge = occ.copy()
    edge[[0, -1], :, :] = 0
    edge[:, [0, -1], :] = 0
    edge[:, :, [0, -1]] = 0
    assert np.array_equal(blender[0], edge)
    if voxels is not None:
        assert occ[1:-1, 1:-1, 1:-1].sum() == voxels[1:-1, 1:-1, 1:-1].sum() > 0
