"""fluidnet_b200/torch7.py: the Torch7 binary reader that brings a model trained with the reference into
this library (SURVEY.md section 8f-2).  A writer for the same format lives here (test-only) so the reader
is exercised without Torch7; the trained 2-D model the reference ships is read when /root/reference is
present and must match the committed fixture (tests/golden/myModel2D_layers.npz)."""
import os

import numpy as np
import pytest

from fluidnet_b200 import torch7
from torch7_writer import GOLD, REF_MODEL, W


def test_reader_round_trip(tmp_path):
    rng = np.random.default_rng(0)
    w1, b1 = rng.standard_normal((4, 3, 3, 3)).astype(np.float32), rng.standard_normal(4).astype(np.float32)
    w2, b2 = rng.standard_normal((1, 4, 1, 1, 1)).astype(np.float32), rng.standard_normal(1).astype(np.float32)
    wr = W()

    def conv2d():
        wr.obj("cudnn.SpatialConvolution", [("weight", lambda: wr.tensor(w1, "torch.CudaTensor", "torch.CudaStorage")),
                                            ("bias", lambda: wr.tensor(b1)), ("nInputPlane", lambda: wr.number(3)),
                                            ("nOutputPlane", lambda: wr.number(4)), ("kH", lambda: wr.number(3)),
                                            ("kW", lambda: wr.number(3)), ("train", lambda: wr.boolean(False))])

    def conv3d():
        wr.obj("cudnn.VolumetricConvolution", [("weight", lambda: wr.tensor(w2)), ("bias", lambda: wr.tensor(b2)),
                                               ("nInputPlane", lambda: wr.number(4)), ("nOutputPlane", lambda: wr.number(1)),
                                               ("kT", lambda: wr.number(1)), ("kH", lambda: wr.number(1)),
                                               ("kW", lambda: wr.number(1))])

    wr.obj("nn.Sequential", [("modules", lambda: wr.table([(1, conv2d), (2, lambda: wr.obj("nn.ReLU", [("inf", lambda: wr.number(float("inf")))])),
                                                            (3, conv3d)])),
                             ("name", lambda: wr.string("net"))])
    path = tmp_path / "net.t7"
    path.write_bytes(bytes(wr.b))
    model = torch7.load(str(path))
    assert model.cls == "nn.Sequential" and model["name"] == "net"
    assert model["modules"][2]["inf"] == float("inf")
    layers = torch7.conv_layers(model)
    assert [w.shape for w, _ in layers] == [(4, 3, 1, 3, 3), (1, 4, 1, 1, 1)]
    assert np.array_equal(layers[0][0].reshape(w1.shape), w1) and np.array_equal(layers[0][1], b1)
    assert np.array_equal(layers[1][0], w2) and np.array_equal(layers[1][1], b2)


def test_back_references(tmp_path):
    wr = W()
    wr.table([("a", lambda: wr.table([(1, lambda: wr.number(7))])), ("b", lambda: wr.backref_table(2))])
    path = tmp_path / "t.t7"
    path.write_bytes(bytes(wr.b))
    t = torch7.load(str(path))
    assert t["a"] is t["b"] and t["a"][1] == 7


@pytest.mark.skipif(not os.path.exists(REF_MODEL), reason="/root/reference not present")
def test_shipped_2d_model_matches_fixture():
    """The reference's trained model (nngraph gModule of cudnn.SpatialConvolution layers): 'default' 2-D
    architecture of torch/lib/model.lua:179-186, and the same numbers as the committed fixture."""
    ref = torch7.load_reference_model(REF_MODEL)
    assert ref["is3D"] is False and ref["mconf"]["modelType"] == "default"
    assert [(w.shape[1], w.shape[0], w.shape[4]) for w, _ in ref["layers"]] == \
        [(3, 16, 3), (16, 16, 3), (16, 16, 3), (16, 16, 3), (16, 1, 1)]
    z = np.load(GOLD)
    assert int(z["n_layers"]) == len(ref["layers"])
    for i, (w, b) in enumerate(ref["layers"]):
        assert np.array_equal(z["w%d" % i], w) and np.array_equal(z["b%d" % i], b)
