"""Dumps what the projection network's drivers compute on seeded inputs, for `cmp` between two builds of the library
(TFL_LIB_PATH selects the build): p and U of tfl_cnn_project in every mode each model takes, p, U and density after
three fused steps where the fused step applies, and a single-rank tfl_slab_sim_step with a 2-bank model.

    TFL_LIB_PATH=... python tests/dbg_forward_dump.py OUTDIR"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    import torch
    from fluidnet_b200 import simulate, synth
    from fluidnet_b200.slab import NativeSlabSimulator
    from fluidnet_b200.model import ProjectionModel
    from scenes import banks, fields_with_random_p, plume_batch, step_mconf

    out = sys.argv[1]
    os.makedirs(out, exist_ok=True)

    def save(name, t):
        np.save(os.path.join(out, name + ".npy"), t.cpu().numpy() if hasattr(t, "cpu") else t)

    skip = {"inputChannels": {"UDiv": True}, "addPressureSkip": True}
    models = [("default", True, {}, (16, 16, 16)), 
              ("mres3-concat", True, {"banks": banks(3, "concat", "mres")}, (16, 16, 16)),
              ("mres3-add", True, {"banks": banks(3, "add", "mres")}, (16, 16, 16)),
              ("dilate2", True, {"banks": banks(2, "concat", "dilate")}, (15, 16, 15)),
              ("bn-batch", True, {"batch_norm": {"train": True}}, (16, 16, 16)),
              ("bn-running", True, {"batch_norm": {"train": False}}, (16, 16, 16)),
              ("udiv-skip", True, {"inputs": skip}, (16, 16, 16)), ("tog", True, {"model_type": "tog"}, (16, 16, 16)),
              ("yang", True, {"model_type": "yang"}, (16, 16, 16)), ("default2d", False, {}, (1, 32, 32))]
    for name, is3d, kw, (nz, ny, nx) in models:
        mnp = synth.make_model(is3d, **kw)
        f = {k: torch.from_numpy(v).cuda() for k, v in fields_with_random_p(nz, ny, nx, is3d).items()}
        for mode in ("fp32", "tf32", "tf32x3"):
            try:
                gm = ProjectionModel.from_model(mnp)
                gm.set_mode(mode)
            except Exception:       # the model does not take this mode
                assert mode != "fp32"
                continue
            p, U = gm.forward((f["pDiv"], f["UDiv"], f["flags"]))
            save("%s-%s-p" % (name, mode), p)
            save("%s-%s-U" % (name, mode), U)
    for name, bk in (("default", None), ("mres2", banks(2, "concat", "mres")), ("mres3-add", banks(3, "add", "mres"))):
        batch, mconf, mnp = plume_batch(32, inflow=32 / 128.0 * 4), step_mconf(32), synth.make_model(True, banks=bk)
        gm = ProjectionModel.from_model(mnp)
        gm.set_mode("tf32x3")
        gb = {k: torch.from_numpy(v).cuda() for k, v in batch.items()}
        for _ in range(3):
            simulate.simulate_fused(None, mconf, gb, gm)
        for k in ("pDiv", "UDiv", "density"):
            save("step-%s-%s" % (name, k), gb[k])
    bk = banks(2, "concat")
    batch, mconf, mnp = plume_batch(32, inflow=32 / 128.0 * 4), step_mconf(32), synth.make_model(True, banks=bk)
    tb = {k: torch.from_numpy(v) for k, v in batch.items()}
    sim = NativeSlabSimulator(tb, mconf, mnp["layers"], torch.device("cuda", 0), rank=0, world=1, banks=bk)
    for _ in range(3):
        sim.step()
    for k in ("pDiv", "UDiv", "density"):
        save("slab-mres2-%s" % k, sim.gather(k))
    sim.close()
    print("dumped %d arrays to %s" % (len(os.listdir(out)), out))


if __name__ == "__main__":
    main()
