"""ProjectionModel.from_model: every key of a model dict reaches the constructor, and a key it does not know raises
(the constructor is replaced by a recorder, so no device is needed)."""
import pytest

from fluidnet_b200 import synth
from fluidnet_b200.model import ProjectionModel


@pytest.fixture
def recorded(monkeypatch):
    calls = []
    monkeypatch.setattr(ProjectionModel, "__init__", lambda self, *a, **kw: calls.append((a, kw)))
    return calls


def test_every_key_reaches_the_constructor(recorded):
    m = synth.make_model(True, model_type="tog",
                         banks={"num": 2, "split_stage": 1, "join_stage": 3, "aggregate": "add", "type": "dilate"},
                         inputs={"inputChannels": {"UDiv": True}, "normalizeInputChan": "div", "addPressureSkip": True},
                         batch_norm={"train": False})
    m["nonlinType"] = "relu6"
    m["poolType"] = "max"
    assert set(m) == set(ProjectionModel.MODEL_KEYS)
    ProjectionModel.from_model(m, device="cuda:1", normalizeInputThreshold=0.25)
    (args, kw), = recorded
    assert args == (m["layers"], True)
    assert kw == dict(device="cuda:1", normalizeInputThreshold=0.25, pool=m["pool"], up=m["up"], poolType="max",
                      nonlinType="relu6", banks=m["banks"], batchNorm=m["batchNorm"], **m["inputs"])


def test_a_plain_model_passes_only_what_it_holds(recorded):
    m = synth.make_model(False)
    ProjectionModel.from_model(m)
    assert recorded == [((m["layers"], False), dict(device=None, normalizeInputThreshold=1e-5))]


def test_an_unknown_key_raises(recorded):
    m = dict(synth.make_model(True), banksNum=2)
    with pytest.raises(ValueError, match="banksNum"):
        ProjectionModel.from_model(m)
    assert recorded == []
