"""Import of reference models through the mconf and the nngraph annotations (fluidnet_b200/torch7.py
graph_stages / model_options / check_stages): banked graphs, the options the library refuses by name, and the
shipped 2-D model.  Torch7 files are written with the test writer of tests/test_torch7_reader.py."""
import os

import numpy as np
import pytest

from fluidnet_b200 import synth, torch7
from test_torch7_reader import GOLD, REF_MODEL, W


def write_graph(path, nodes, is3d):
    """An nn.gModule whose forwardnodes hold `nodes` = [(module class, fields or None, annotation or None)]."""
    wr = W()

    def conv(w, b):
        cls = "cudnn.VolumetricConvolution" if is3d else "cudnn.SpatialConvolution"
        k = w.shape[-1]
        items = [("weight", lambda: wr.tensor(w if is3d else w[:, :, 0])), ("bias", lambda: wr.tensor(b)),
                 ("nInputPlane", lambda: wr.number(w.shape[1])), ("nOutputPlane", lambda: wr.number(w.shape[0])),
                 ("kH", lambda: wr.number(k)), ("kW", lambda: wr.number(k))]
        if is3d:
            items.append(("kT", lambda: wr.number(k)))
        return lambda: wr.obj(cls, items)

    def node(cls, fields, name):
        mod = conv(*fields) if fields is not None else (lambda: wr.obj(cls, [("train", lambda: wr.boolean(False))]))
        data = [("module", mod)]
        if name:
            data.append(("annotations", lambda: wr.table([("name", lambda: wr.string(name))])))
        return lambda: wr.obj("nngraph.Node", [("data", lambda: wr.table(data))])

    items = [(i + 1, node(*n)) for i, n in enumerate(nodes)]
    wr.obj("nn.gModule", [("forwardnodes", lambda: wr.table(items))])
    path.write_bytes(bytes(wr.b))


def graph_nodes(model, extra=()):
    """The nodes of lib/model.lua:27-401 for a synth.make_model model (with banks), in forward order."""
    nodes = [("nn.Identity", None, "input"), ("tfluids.SetWallBcs", None, None), ("nn.JoinTable", None, "pModelInput")]
    nl = len(model["layers"])
    for s, layer in enumerate(model["layers"], start=1):
        convs = layer if isinstance(layer, list) else [layer]
        for bank, (w, b) in enumerate(convs, start=1):
            nodes.append((None, (w, b), None if s == nl else "Bank %d: conv stage %d" % (bank, s)))
            if s < nl:
                nodes.append(("nn.ReLU", None, "Bank %d: non-linearity" % bank))
    nodes += list(extra)
    nodes += [("tfluids.VelocityUpdate", None, "UPred"), ("tfluids.SetWallBcs", None, "U")]
    return nodes


def mconf_of(is3d, **kw):
    m = {"is3D": is3d, "modelType": "default", "nonlinType": "relu", "poolType": "avg", "banksNum": 1,
         "banksSplitStage": 1, "banksJoinStage": 3, "banksAggregateMethod": "concat", "banksType": "mres",
         "banksWeightShare": False, "addBatchNorm": False, "addPressureSkip": False, "normalizeInput": True,
         "normalizeInputFunc": "std", "normalizeInputChan": "UDiv", "normalizeInputThreshold": 1e-5,
         "inputChannels": {"pDiv": True, "div": True, "flags": True, "UDiv": False}}
    m.update(kw)
    return m


@pytest.mark.parametrize("is3d,num,agg", [(True, 2, "concat"), (True, 3, "add"), (False, 2, "concat")])
def test_banked_file_loads_to_the_same_layers(tmp_path, is3d, num, agg):
    model = synth.make_model(is3d, banks={"num": num, "split_stage": 1, "join_stage": 3, "aggregate": agg})
    write_graph(tmp_path / "net", graph_nodes(model), is3d)
    mconf = mconf_of(is3d, banksNum=num, banksAggregateMethod=agg)
    stages = torch7.graph_stages(torch7.load(str(tmp_path / "net")))
    opts = torch7.model_options(mconf)
    torch7.check_stages(stages, mconf, opts)
    assert opts["banks"] == {"num": num, "split_stage": 1, "join_stage": 3, "aggregate": agg}
    assert len(stages) == len(model["layers"])
    for got, want in zip(stages, model["layers"]):
        got = got if isinstance(got, list) else [got]
        want = want if isinstance(want, list) else [want]
        assert len(got) == len(want)
        for (gw, gb), (ww, wb) in zip(got, want):
            assert np.array_equal(gw, ww) and np.array_equal(gb, wb)


@pytest.mark.parametrize("key,value,name", [
    ("addBatchNorm", True, "addBatchNorm"), ("addPressureSkip", True, "addPressureSkip"),
    ("nonlinType", "relu6", "nonlinType"), ("normalizeInput", False, "normalizeInput"),
    ("normalizeInputFunc", "norm", "normalizeInputFunc"), ("normalizeInputChan", "U", "normalizeInputChan"),
    ("inputChannels", {"pDiv": True, "div": True, "flags": True, "UDiv": True}, "inputChannels"),
    ("banksType", "dilate", "banksType"), ("banksWeightShare", True, "banksWeightShare"),
])
def test_unsupported_mconf_options_are_refused_by_name(key, value, name):
    mconf = mconf_of(True, banksNum=2, **{key: value})
    with pytest.raises(ValueError, match=name):
        torch7.model_options(mconf)


@pytest.mark.parametrize("cls", ["cudnn.SpatialBatchNormalization", "nn.CMulTable", "nn.SpatialDilatedConvolution"])
def test_unsupported_modules_are_refused_by_name(tmp_path, cls):
    model = synth.make_model(False)
    write_graph(tmp_path / "net", graph_nodes(model, extra=[(cls, None, None)]), False)
    with pytest.raises(ValueError, match=cls):
        torch7.graph_stages(torch7.load(str(tmp_path / "net")))


def test_low_rank_sequential_is_refused(tmp_path):
    wr = W()
    w, b = synth.make_model(False)["layers"][0]
    conv = lambda: wr.obj("cudnn.SpatialConvolution", [("weight", lambda: wr.tensor(w[:, :, 0])), ("bias", lambda: wr.tensor(b)),
                                                       ("nInputPlane", lambda: wr.number(3)), ("nOutputPlane", lambda: wr.number(16)),
                                                       ("kH", lambda: wr.number(3)), ("kW", lambda: wr.number(3))])
    seq = lambda: wr.obj("nn.Sequential", [("modules", lambda: wr.table([(1, conv)]))])
    node = lambda: wr.obj("nngraph.Node", [("data", lambda: wr.table([("module", seq)]))])
    wr.obj("nn.gModule", [("forwardnodes", lambda: wr.table([(1, node)]))])
    (tmp_path / "net").write_bytes(bytes(wr.b))
    with pytest.raises(ValueError, match="nn.Sequential"):
        torch7.graph_stages(torch7.load(str(tmp_path / "net")))


def test_yang_mconf_builds_a_sigmoid_model():
    opts = torch7.model_options(mconf_of(True, modelType="yang", nonlinType="sigmoid"))
    assert opts["nonlinType"] == "sigmoid" and opts["pool"] == [1] * 4 and "banks" not in opts
    tog = torch7.model_options(mconf_of(False, modelType="tog", poolType="max"))
    assert tog["pool"] == [2, 1, 1, 1, 1, 1, 1] and tog["up"] == [1, 1, 1, 1, 1, 1, 2] and tog["poolType"] == "max"


def test_shape_mismatch_is_refused(tmp_path):
    model = synth.make_model(True, banks={"num": 2, "split_stage": 1, "join_stage": 3, "aggregate": "add"})
    write_graph(tmp_path / "net", graph_nodes(model), True)
    stages = torch7.graph_stages(torch7.load(str(tmp_path / "net")))
    mconf = mconf_of(True, banksNum=2, banksAggregateMethod="concat")        # concat needs 16 channels at stage 3
    with pytest.raises(ValueError, match="stage 3"):
        torch7.check_stages(stages, mconf, torch7.model_options(mconf))
    mconf = mconf_of(True, banksNum=3, banksAggregateMethod="add")
    with pytest.raises(ValueError, match="banks"):
        torch7.check_stages(stages, mconf, torch7.model_options(mconf))


@pytest.mark.skipif(not os.path.exists(REF_MODEL), reason="the reference's shipped model is not present")
def test_shipped_2d_model_stages_match_fixture():
    """The shipped myModel2D's annotations ("Bank 1: conv stage 1..4" and one unannotated final convolution) give
    the same five layers as the committed fixture, and its mconf the single-bank 'default' graph."""
    ref = torch7.load_reference_model(REF_MODEL)
    opts = torch7.model_options(ref["mconf"])
    stages = torch7.graph_stages(ref["model"])
    torch7.check_stages(stages, ref["mconf"], opts)
    assert "banks" not in opts and opts["nonlinType"] == "relu" and opts["pool"] == [1] * 5
    z = np.load(GOLD)
    assert int(z["n_layers"]) == len(stages)
    for i, (w, b) in enumerate(stages):
        assert np.array_equal(z["w%d" % i], w) and np.array_equal(z["b%d" % i], b)


def test_missing_stage_is_refused(tmp_path):
    """A stage below the highest annotated one with no convolution at all is named, not an IndexError."""
    model = synth.make_model(False)
    nodes = [n for n in graph_nodes(model) if n[2] != "Bank 1: conv stage 2"]
    write_graph(tmp_path / "net", nodes, False)
    with pytest.raises(ValueError, match="stage 2"):
        torch7.graph_stages(torch7.load(str(tmp_path / "net")))
