"""Import of addBatchNorm / nonlinType 'relu6' reference models (fluidnet_b200/torch7.py batch_norm_layers,
graph_stages(batchnorm=True), model_options(batchnorm=True, relu6=True)): nn and cudnn, Spatial and Volumetric
modules, affine on and off, train true and false, banks of both types, BN nodes assigned through the graph's edges
with banks interleaved in forwardnodes, and every refusal by name.  Torch7 files are written with the test writer of
tests/test_torch7_reader.py, nngraph nodes with their `children` edges."""
import numpy as np
import pytest

from fluidnet_b200 import synth, torch7
from torch7_writer import bn_graph, mconf_for, mconf_of, write_bn_graph


def load_bn(tmp_path, model, is3d, **kw):
    write_bn_graph(tmp_path / "net", bn_graph(model, is3d, **kw), is3d)
    return torch7.load(str(tmp_path / "net"))


CASES = {   # (is3d, banks, cudnn / affine, train, interleave)
    "3d-cudnn-train": (True, None, True, True, False),
    "3d-nn-eval": (True, None, False, False, False),
    "2d-cudnn-eval": (False, None, True, False, False),
    "2d-nn-train": (False, None, False, True, False),
    "3d-mres-n3-concat-interleaved": (True, {"num": 3, "split_stage": 1, "join_stage": 3, "aggregate": "concat"},
                                      True, True, True),
    "3d-dilate-n2-add": (True, {"num": 2, "split_stage": 1, "join_stage": 3, "aggregate": "add", "type": "dilate"},
                         False, False, False),
    "2d-mres-n2-add-interleaved": (False, {"num": 2, "split_stage": 2, "join_stage": 4, "aggregate": "add"},
                                   True, False, True),
}


@pytest.mark.parametrize("case", list(CASES))
def test_bn_file_loads_to_the_same_parameters(tmp_path, case):
    is3d, bk, cudnn, train, inter = CASES[case]
    model = synth.make_model(is3d, banks=bk, batch_norm={"train": train, "affine": cudnn})
    net = load_bn(tmp_path, model, is3d, cudnn=cudnn, train=train, interleave=inter)
    mconf = mconf_for(is3d, bk, cudnn)
    bn = torch7.batch_norm_layers(net)
    opts = torch7.model_options(mconf, inputs=True, dilate=True, batchnorm=True, bn=bn)
    stages = torch7.graph_stages(net, dilate=False, batchnorm=True)
    torch7.check_stages(stages, mconf, opts)
    assert opts["batchNorm"]["train"] is train
    for got, want in zip(opts["batchNorm"]["layers"], model["batchNorm"]["layers"]):
        got = got if isinstance(got, list) else [got]
        want = want if isinstance(want, list) else [want]
        assert len(got) == len(want)
        for g, w in zip(got, want):
            for k in ("weight", "bias", "running_mean", "running_var"):
                assert (g[k] is None) == (w[k] is None), k
                if w[k] is not None:
                    assert np.array_equal(g[k], w[k]), k
            assert g["eps"] == w["eps"]


def test_relu6_model_loads(tmp_path):
    model = synth.make_model(True, batch_norm={"train": True})
    net = load_bn(tmp_path, model, True, nonlin="nn.ReLU6")
    opts = torch7.model_options(mconf_for(True, None, True, nonlinType="relu6"), batchnorm=True, relu6=True,
                                bn=torch7.batch_norm_layers(net))
    assert opts["nonlinType"] == "relu6"
    torch7.graph_stages(net, batchnorm=True)


def test_refusals_by_name(tmp_path):
    bk = {"num": 2, "split_stage": 1, "join_stage": 3, "aggregate": "concat"}
    model = synth.make_model(True, banks=bk, batch_norm={"train": True})
    with pytest.raises(ValueError, match="stage 2 bank 2 has no batch normalization"):
        torch7.batch_norm_layers(load_bn(tmp_path, model, True, drop=(2, 2)))
    with pytest.raises(ValueError, match="not placed after a stage"):
        torch7.batch_norm_layers(load_bn(tmp_path, model, True, misplace=True))
    with pytest.raises(ValueError, match="differ in their train flag"):
        torch7.batch_norm_layers(load_bn(tmp_path, model, True, train_of=(1, 2)))
    with pytest.raises(ValueError, match="running_std without running_var"):
        torch7.batch_norm_layers(load_bn(tmp_path, model, True, old_format=True))
    with pytest.raises(ValueError, match="9 channels"):
        torch7.batch_norm_layers(load_bn(tmp_path, model, True, channels=(2, 1)))
    net = load_bn(tmp_path, model, True)
    bn = torch7.batch_norm_layers(net)
    with pytest.raises(ValueError, match="batchNormAffine"):
        torch7.model_options(mconf_for(True, bk, False), batchnorm=True, bn=bn)
    with pytest.raises(ValueError, match="batchNormEps"):
        torch7.model_options(mconf_for(True, bk, True, batchNormEps=1e-3), batchnorm=True, bn=bn)
    with pytest.raises(ValueError, match="addBatchNorm"):
        torch7.model_options(mconf_for(True, bk, True), batchnorm=True)       # no modules given


def test_calls_without_the_keywords_still_refuse(tmp_path):
    model = synth.make_model(True, batch_norm={"train": True})
    net = load_bn(tmp_path, model, True)
    with pytest.raises(ValueError, match="BatchNormalization"):
        torch7.graph_stages(net)
    with pytest.raises(ValueError, match="addBatchNorm"):
        torch7.model_options(mconf_for(True, None, True))
    with pytest.raises(ValueError, match="nonlinType"):
        torch7.model_options(mconf_of(True, nonlinType="relu6"), batchnorm=True)
