"""Import of reference models trained with the input-block options of lib/model.lua:27-150 and :357-387
(inputChannels, normalizeInput, normalizeInputFunc, normalizeInputChan, addPressureSkip): synthetic Torch7 files
through the steps of ProjectionModel.from_reference_file (model_options(mconf, inputs=True), graph_stages,
check_stages), every combination the reference cannot build refused naming its key, and the default
model_options(mconf) still refusing the keys it would drop."""
import numpy as np
import pytest

from fluidnet_b200 import synth, torch7
from torch7_writer import graph_nodes, mconf_of, write_graph

ALL = {"pDiv": True, "UDiv": True, "div": True, "flags": True}
U_ONLY = {"pDiv": False, "UDiv": True, "div": False, "flags": True}
DIV_ONLY = {"pDiv": False, "UDiv": False, "div": True, "flags": True}


def load_like_from_reference_file(tmp_path, model, mconf):
    write_graph(tmp_path / "net", graph_nodes(model), model["is3D"])
    opts = torch7.model_options(mconf, inputs=True)
    stages = torch7.graph_stages(torch7.load(str(tmp_path / "net")))
    torch7.check_stages(stages, mconf, opts)
    return stages, opts


@pytest.mark.parametrize("is3d,model_type,keys", [
    (True, "default", dict(inputChannels=ALL, addPressureSkip=True)),
    (True, "default", dict(inputChannels=U_ONLY, normalizeInputFunc="norm")),
    (False, "default", dict(inputChannels=ALL, normalizeInputChan="div", addPressureSkip=True)),
    (False, "default", dict(inputChannels=DIV_ONLY, normalizeInputChan="pDiv")),
    (True, "default", dict(normalizeInput=False)),
    (True, "yang", dict(nonlinType="sigmoid", addPressureSkip=True, normalizeInputFunc="norm")),
    (False, "tog", dict(inputChannels=ALL)),
], ids=["3d-all-skip", "3d-U-norm", "2d-all-divchan-skip", "2d-div-pchan", "3d-unnormalized", "3d-yang-skip",
        "2d-tog-all"])
def test_file_loads_with_its_input_block(tmp_path, is3d, model_type, keys):
    mconf = mconf_of(is3d, modelType=model_type, **keys)
    want_inputs = torch7.input_options(mconf)
    model = synth.make_model(is3d, model_type=model_type, inputs=want_inputs)
    stages, opts = load_like_from_reference_file(tmp_path, model, mconf)
    for k, v in want_inputs.items():
        assert opts[k] == v
    ch = want_inputs["inputChannels"]
    assert stages[0][0].shape[1] == ch["pDiv"] + (3 if is3d else 2) * ch["UDiv"] + ch["div"] + 1
    assert stages[-1][0].shape[1] == stages[-2][0].shape[0] + bool(keys.get("addPressureSkip"))
    for (gw, gb), (ww, wb) in zip(stages, model["layers"]):
        assert np.array_equal(gw, ww) and np.array_equal(gb, wb)


def test_default_mconf_gives_the_default_block():
    opts = torch7.model_options(mconf_of(True), inputs=True)
    assert opts["inputChannels"] == {"pDiv": True, "UDiv": False, "div": True, "flags": True}
    assert (opts["normalizeInput"], opts["normalizeInputFunc"], opts["normalizeInputChan"], opts["addPressureSkip"]) \
        == (True, "std", "UDiv", False)


def test_file_whose_first_layer_misses_a_channel_is_refused(tmp_path):
    mconf = mconf_of(True, inputChannels=ALL)
    model = synth.make_model(True)                     # 3 input channels, the mconf gives 6
    with pytest.raises(ValueError, match="stage 1"):
        load_like_from_reference_file(tmp_path, model, mconf)


def test_file_without_the_skip_channel_is_refused(tmp_path):
    mconf = mconf_of(True, addPressureSkip=True)
    model = synth.make_model(True)
    with pytest.raises(ValueError, match="stage 5"):
        load_like_from_reference_file(tmp_path, model, mconf)


@pytest.mark.parametrize("keys,name,why", [
    (dict(inputChannels={"pDiv": True, "div": True, "flags": False}), "inputChannels", "flags on input"),
    (dict(inputChannels={"pDiv": False, "div": False, "UDiv": False, "flags": True}), "inputChannels",
     "any \\(U, div or p\\)"),
    (dict(inputChannels={"pDiv": True, "div": False, "UDiv": False, "flags": True}), "inputChannels", "VelocityUpdate"),
    (dict(normalizeInputFunc="l1"), "normalizeInputFunc", "Incorrect normalize input function"),
    (dict(normalizeInputChan="uDiv"), "normalizeInputChan", "Incorrect normalize input channel"),
    (dict(normalizeInputChan="div", inputChannels=U_ONLY), "normalizeInputChan", "needs inputChannels.div"),
    (dict(modelType="yang", nonlinType="sigmoid", inputChannels=ALL), "inputChannels", "must not have UDiv"),
    (dict(modelType="yang", nonlinType="sigmoid", inputChannels=DIV_ONLY), "inputChannels", "must have pDiv"),
    (dict(modelType="tog", addPressureSkip=True), "addPressureSkip", "tog"),
], ids=["no-flags", "no-field", "no-U-for-update", "func", "chan", "div-chan-without-div", "yang-U", "yang-no-p",
        "tog-skip"])
def test_unbuildable_blocks_are_refused_by_key(keys, name, why):
    mconf = mconf_of(True, **keys)
    with pytest.raises(ValueError, match="%s: .*%s" % (name, why)):
        torch7.model_options(mconf, inputs=True)


@pytest.mark.parametrize("key,value", [("addPressureSkip", True), ("inputChannels", ALL), ("normalizeInput", False),
                                       ("normalizeInputFunc", "norm"), ("normalizeInputChan", "pDiv")])
def test_default_call_still_refuses_the_keys(key, value):
    with pytest.raises(ValueError, match=key):
        torch7.model_options(mconf_of(True, **{key: value}))
