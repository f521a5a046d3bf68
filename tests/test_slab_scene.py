"""The demo scene's z-slab mode on the host (fluidnet_b200/scene.py): its refusals come before any rank touches a GPU,
its margin default, and the files it writes are named and headed as the single-GPU scene's."""
import os

import numpy as np
import pytest

from fluidnet_b200 import formats, scene


def test_pcg_is_refused_by_name_before_anything_runs(monkeypatch):
    with pytest.raises(ValueError, match="simMethod 'pcg' does not run on z-slabs"):
        scene.check_slab_args(128, "pcg", 1, None)
    with pytest.raises(ValueError, match="simMethod 'pcg' does not run on z-slabs"):
        scene.run(32, "plume", "pcg", slabs=True, world=1, rank=0, log=lambda *a: None)
    monkeypatch.setenv("WORLD_SIZE", "2")             # torchrun with two processes implies --slabs
    with pytest.raises(ValueError, match="simMethod 'pcg' does not run on z-slabs"):
        scene.main(["--res", "64", "--sim-method", "pcg"])


def test_margin_default_and_floor():
    assert scene.check_slab_args(256, "jacobi", 8, None) == scene.SLAB_MARGIN == 5
    assert scene.check_slab_args(256, "convnet", 8, 5) == 5
    with pytest.raises(ValueError, match="--margin must be >= 2"):
        scene.check_slab_args(256, "jacobi", 8, 1)


@pytest.mark.parametrize("res,world,margin", [(32, 8, None), (64, 8, 4), (256, 64, 2), (512, 32, 8), (256, 32, None)])
def test_slabs_thinner_than_the_halo_are_refused_before_any_rank_starts(res, world, margin, tmp_path):
    halo = 2 * (margin or scene.SLAB_MARGIN) + 2
    assert res // world < halo
    with pytest.raises(ValueError, match="thinner than the halo of %d" % halo):
        scene.check_slab_args(res, "jacobi", world, margin)
    with pytest.raises(ValueError, match="thinner than the halo"):
        scene.run(res, "plume", "jacobi", out_dir=str(tmp_path), slabs=True, margin=margin, world=world, rank=0,
                  log=lambda *a: None)
    assert not os.listdir(str(tmp_path))                # refused before a file or directory was made
    assert scene.check_slab_args(res, "jacobi", 1, margin) == (margin or scene.SLAB_MARGIN)   # one rank: no halo


def test_main_refuses_thin_slabs_under_torchrun(monkeypatch):
    monkeypatch.setenv("WORLD_SIZE", "32")
    monkeypatch.setenv("RANK", "3")
    with pytest.raises(ValueError, match="32 ranks give slabs of 4 planes"):
        scene.main(["--res", "128", "--sim-method", "jacobi"])
    assert scene.launcher_world() == (3, 32, 0)


@pytest.mark.parametrize("which,model_name,density_file", [("plume", "none", None), ("arch", "myModel3D", None),
                                                          ("bunny", "synthetic", "elsewhere/d.vbox")])
def test_slab_files_are_named_as_the_single_gpu_scene(which, model_name, density_file):
    paths = scene.scene_paths(None, which, model_name, 0.1, density_file)
    assert paths["density"] == (density_file or os.path.join(scene.SCENES[which], scene.density_filename(model_name, 0.1)))
    assert paths["density"].endswith("_dt0.1.vbox") or density_file
    assert paths["geom"] == os.path.join(scene.SCENES[which], "geom_output.vbox")
    assert paths["geom_blender"] == os.path.join(scene.SCENES[which], "geom_output_blender.vbox")


def test_slab_density_header_is_the_single_gpu_scene_header(tmp_path):
    """Both modes open the density file as VboxWriter(path, res, numFrames): the header counts numFrames frames while
    every third is written; a frame packed by the recorder ([nx][ny][nz]) and one written from the grid agree."""
    res, frames = 24, 768
    grid = np.random.default_rng(3).random((1, 1, res, res, res), dtype=np.float32)
    a, b = str(tmp_path / "a.vbox"), str(tmp_path / "b.vbox")
    with formats.VboxWriter(a, res, frames) as w:
        w.write(grid)
    with formats.VboxWriter(b, res, frames) as w:
        w.write_packed(np.ascontiguousarray(grid[0, 0].transpose(2, 1, 0)))
    with open(a, "rb") as f, open(b, "rb") as g:
        ba, bb = f.read(), g.read()
    assert ba == bb and np.frombuffer(ba[:16], np.int32).tolist() == [res, res, res, frames]
