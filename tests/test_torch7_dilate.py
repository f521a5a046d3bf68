"""Import of banksType 'dilate' reference models (fluidnet_b200/torch7.py model_options / graph_stages with
dilate=True): bank i >= 2's convolutions are nn.{Spatial,Volumetric}DilatedConvolution with dilation 2^(i-1), stride 1
and padding 2^(i-1) (k-1)/2 (lib/model_utils.lua:122-146), and they load to the layers synth.make_model draws.  The
default calls keep refusing dilated models (tests/test_torch7_banks.py).  Torch7 files are written with the test
writer of tests/test_torch7_reader.py."""
import numpy as np
import pytest

from fluidnet_b200 import synth, torch7
from test_torch7_banks import mconf_of
from test_torch7_reader import W


def conv_module(wr, w, b, is3d, d=1, pad=None, stride=1):
    """A convolution module: cudnn.{Spatial,Volumetric}Convolution for d = 1, nn.*DilatedConvolution (with the
    fields of torch's nn package) otherwise; pad defaults to d (k-1)/2."""
    k = w.shape[-1]
    pad = d * (k - 1) // 2 if pad is None else pad
    axes = ("T", "W", "H") if is3d else ("W", "H")
    if d == 1:
        cls = "cudnn.VolumetricConvolution" if is3d else "cudnn.SpatialConvolution"
    else:
        cls = "nn.VolumetricDilatedConvolution" if is3d else "nn.SpatialDilatedConvolution"
    items = [("weight", lambda: wr.tensor(w if is3d else w[:, :, 0])), ("bias", lambda: wr.tensor(b)),
             ("nInputPlane", lambda: wr.number(w.shape[1])), ("nOutputPlane", lambda: wr.number(w.shape[0]))]
    for a in axes:
        items += [("k" + a, lambda: wr.number(k)), ("d" + a, lambda: wr.number(stride)),
                  ("pad" + a, lambda: wr.number(pad))]
        if d != 1:
            items.append(("dilation" + a, lambda: wr.number(d)))
    return lambda: wr.obj(cls, items)


def write_dilated(path, model, is3d, dil_of=None, extra=()):
    """The nodes of lib/model.lua:27-401 for a synth.make_model model; bank i's convolution is dilated by
    dil_of(bank, stage) (default: 2^(bank-1), as the reference builds it), with keyword overrides from a dict."""
    wr = W()
    dil_of = dil_of or (lambda bank, stage: {"d": 2 ** (bank - 1)})

    def plain(cls, name):
        data = [("module", lambda: wr.obj(cls, [("train", lambda: wr.boolean(False))]))]
        if name:
            data.append(("annotations", lambda: wr.table([("name", lambda: wr.string(name))])))
        return lambda: wr.obj("nngraph.Node", [("data", lambda: wr.table(data))])

    def conv_node(w, b, name, kw):
        data = [("module", conv_module(wr, w, b, is3d, **kw))]
        if name:
            data.append(("annotations", lambda: wr.table([("name", lambda: wr.string(name))])))
        return lambda: wr.obj("nngraph.Node", [("data", lambda: wr.table(data))])

    nodes = [plain("nn.Identity", "input"), plain("tfluids.SetWallBcs", None), plain("nn.JoinTable", "pModelInput")]
    nl = len(model["layers"])
    for s, layer in enumerate(model["layers"], start=1):
        convs = layer if isinstance(layer, list) else [layer]
        for bank, (w, b) in enumerate(convs, start=1):
            name = None if s == nl else "Bank %d: conv stage %d" % (bank, s)
            kw = dil_of(bank, s) if (s < nl and len(convs) > 1) else {}
            nodes.append(conv_node(w, b, name, kw))
            if s < nl:
                nodes.append(plain("nn.ReLU", "Bank %d: non-linearity" % bank))
    nodes += [plain(*e) for e in extra]
    nodes += [plain("tfluids.VelocityUpdate", "UPred"), plain("tfluids.SetWallBcs", "U")]
    items = [(i + 1, n) for i, n in enumerate(nodes)]
    wr.obj("nn.gModule", [("forwardnodes", lambda: wr.table(items))])
    path.write_bytes(bytes(wr.b))


def dilate(num, agg, s=1, j=3):
    return {"num": num, "split_stage": s, "join_stage": j, "aggregate": agg, "type": "dilate"}


@pytest.mark.parametrize("is3d,num,agg,s,j", [(True, 2, "concat", 1, 3), (True, 3, "add", 1, 3),
                                              (True, 4, "concat", 2, 4), (False, 2, "concat", 1, 3),
                                              (False, 3, "add", 2, 4)])
def test_dilated_file_loads_to_the_same_layers(tmp_path, is3d, num, agg, s, j):
    model = synth.make_model(is3d, banks=dilate(num, agg, s, j))
    write_dilated(tmp_path / "net", model, is3d)
    mconf = mconf_of(is3d, banksNum=num, banksAggregateMethod=agg, banksType="dilate", banksSplitStage=s,
                     banksJoinStage=j)
    stages = torch7.graph_stages(torch7.load(str(tmp_path / "net")), dilate=True)
    opts = torch7.model_options(mconf, dilate=True)
    torch7.check_stages(stages, mconf, opts)
    assert opts["banks"] == dilate(num, agg, s, j)
    assert len(stages) == len(model["layers"])
    for got, want in zip(stages, model["layers"]):
        got = got if isinstance(got, list) else [got]
        want = want if isinstance(want, list) else [want]
        assert len(got) == len(want)
        for (gw, gb), (ww, wb) in zip(got, want):
            assert np.array_equal(gw, ww) and np.array_equal(gb, wb)


def test_default_calls_still_refuse_dilate(tmp_path):
    """Without dilate=True: the mconf key and the dilated modules are refused by name, as before."""
    with pytest.raises(ValueError, match="banksType"):
        torch7.model_options(mconf_of(True, banksNum=2, banksType="dilate"))
    with pytest.raises(ValueError, match="banksType"):
        torch7.model_options(mconf_of(True, banksNum=2, banksType="dilate"), inputs=True)
    model = synth.make_model(True, banks=dilate(2, "concat"))
    write_dilated(tmp_path / "net", model, True)
    with pytest.raises(ValueError, match="nn.VolumetricDilatedConvolution"):
        torch7.graph_stages(torch7.load(str(tmp_path / "net")))


def test_dilate_keyword_keeps_other_options():
    """dilate=True changes nothing for 'mres' or single-bank mconfs (no "type" key), and still refuses unknown types
    and banksWeightShare."""
    m = mconf_of(True, banksNum=2)
    assert torch7.model_options(m, dilate=True) == torch7.model_options(m)
    assert "type" not in torch7.model_options(m, dilate=True)["banks"]
    one = mconf_of(True, banksNum=1, banksType="dilate")
    assert "banks" not in torch7.model_options(one, dilate=True)
    with pytest.raises(ValueError, match="banksType"):
        torch7.model_options(mconf_of(True, banksNum=2, banksType="pyramid"), dilate=True)
    with pytest.raises(ValueError, match="banksWeightShare"):
        torch7.model_options(mconf_of(True, banksNum=2, banksType="dilate", banksWeightShare=True), dilate=True)


@pytest.mark.parametrize("what,dil_of,match", [
    ("undilated bank 2", lambda bank, s: {"d": 1}, "bank 2's convolution .* not a dilated convolution"),
    ("bank 3 at dilation 2", lambda bank, s: {"d": 2 if bank == 3 else 2 ** (bank - 1)}, "bank 3's convolution"),
    ("wrong padding", lambda bank, s: {"d": 2 ** (bank - 1), "pad": 1}, "pad"),
    ("stride 2", lambda bank, s: {"d": 2 ** (bank - 1), "stride": 2}, "stride"),
])
def test_wrong_dilation_is_refused(tmp_path, what, dil_of, match):
    model = synth.make_model(True, banks=dilate(3, "add"))
    write_dilated(tmp_path / "net", model, True, dil_of=dil_of)
    with pytest.raises(ValueError, match=match):
        torch7.graph_stages(torch7.load(str(tmp_path / "net")), dilate=True)


def test_dilated_bank_one_and_final_are_refused(tmp_path):
    model = synth.make_model(False, banks=dilate(2, "concat"))
    write_dilated(tmp_path / "net", model, False, dil_of=lambda bank, s: {"d": 2 if bank == 1 else 2})
    with pytest.raises(ValueError, match="bank 1's convolution is nn.SpatialDilatedConvolution"):
        torch7.graph_stages(torch7.load(str(tmp_path / "net")), dilate=True)


def test_mres_file_with_dilated_modules_is_refused(tmp_path):
    """from_reference_file reads an 'mres' mconf with graph_stages(model, dilate=False): a dilated module is named."""
    model = synth.make_model(True, banks=dilate(2, "add"))
    write_dilated(tmp_path / "net", model, True)
    opts = torch7.model_options(mconf_of(True, banksNum=2, banksAggregateMethod="add"), inputs=True, dilate=True)
    assert "type" not in opts["banks"]
    with pytest.raises(ValueError, match="nn.VolumetricDilatedConvolution"):
        torch7.graph_stages(torch7.load(str(tmp_path / "net")), dilate=opts["banks"].get("type") == "dilate")
