"""Import of addBatchNorm / nonlinType 'relu6' reference models (fluidnet_b200/torch7.py batch_norm_layers,
graph_stages(batchnorm=True), model_options(batchnorm=True, relu6=True)): nn and cudnn, Spatial and Volumetric
modules, affine on and off, train true and false, banks of both types, BN nodes assigned through the graph's edges
with banks interleaved in forwardnodes, and every refusal by name.  Torch7 files are written with the test writer of
tests/test_torch7_reader.py, nngraph nodes with their `children` edges."""
import numpy as np
import pytest

from fluidnet_b200 import synth, torch7
from test_torch7_banks import mconf_of
from test_torch7_reader import W


def bn_graph(model, is3d, nonlin="nn.ReLU", interleave=False, cudnn=True, train=True, old_format=False,
             drop=None, misplace=False, channels=None, train_of=None):
    """lib/model.lua's nodes for a synth.make_model(batch_norm=...) model: per stage and bank conv -> non-linearity ->
    BN (each node's child the next), the banks' chains one after another or interleaved node by node in
    forwardnodes.  Returns [(class, fields, annotation, [child indices])]."""
    nodes = [("nn.Identity", None, "input", [1]), ("nn.JoinTable", None, "pModelInput", [])]
    prev = [1]          # the nodes feeding the next stage
    nl = len(model["layers"])
    bnl = model["batchNorm"]["layers"]
    kind = ("cudnn." if cudnn else "nn.") + ("Volumetric" if is3d else "Spatial") + "BatchNormalization"
    for s, layer in enumerate(model["layers"], start=1):
        convs = layer if isinstance(layer, list) else [layer]
        if s == nl:
            i = len(nodes)
            nodes.append((None, convs[0], None, []))
            for p in prev:
                nodes[p][3].append(i)
            break
        bns = bnl[s - 1] if isinstance(bnl[s - 1], list) else [bnl[s - 1]]
        chains = []
        for bank, ((w, b), e) in enumerate(zip(convs, bns), start=1):
            fields = dict(e)
            if channels is not None and (s, bank) == channels:
                fields["running_mean"] = np.zeros(len(e["running_mean"]) + 1, np.float32)
            tr = train if train_of is None or (s, bank) != train_of else not train
            chains.append([(None, (w, b), "Bank %d: conv stage %d" % (bank, s)),
                           (nonlin, None, "Bank %d: non-linearity" % bank),
                           (kind, ("bn", fields, tr, old_format), None)])
        if drop is not None:
            chains = [c if (s, k + 1) != drop else c[:2] for k, c in enumerate(chains)]
        order = [n for step in zip(*[c + [None] * (3 - len(c)) for c in chains]) for n in step if n is not None] \
            if interleave else [n for c in chains for n in c]
        idx = {}
        for n in order:
            idx[id(n)] = len(nodes)
            nodes.append((n[0], n[1], n[2], []))
        ends = []
        for c in chains:
            ids = [idx[id(n)] for n in c]
            for a, b in zip(ids, ids[1:]):
                nodes[a][3].append(b)
            for p in prev:
                nodes[p][3].append(ids[0])
            ends.append(ids[-1])
        if misplace and s == 1:
            # a BN node fed by the join of the banks, not by a stage's non-linearity
            j = len(nodes)
            nodes.append(("nn.JoinTable", None, None, []))
            k = len(nodes)
            nodes.append((kind, ("bn", dict(bns[0]), train, False), None, []))
            nodes[j][3].append(k)
            for e_ in ends:
                nodes[e_][3].append(j)
        prev = ends
    return nodes


def write_bn_graph(path, nodes, is3d):
    wr = W()
    written = {}

    def conv(w, b):
        cls = "cudnn.VolumetricConvolution" if is3d else "cudnn.SpatialConvolution"
        k = w.shape[-1]
        items = [("weight", lambda: wr.tensor(w if is3d else w[:, :, 0])), ("bias", lambda: wr.tensor(b)),
                 ("nInputPlane", lambda: wr.number(w.shape[1])), ("nOutputPlane", lambda: wr.number(w.shape[0])),
                 ("kH", lambda: wr.number(k)), ("kW", lambda: wr.number(k))]
        if is3d:
            items.append(("kT", lambda: wr.number(k)))
        return lambda: wr.obj(cls, items)

    def bn_mod(cls, fields, train, old):
        items = [("running_mean", lambda: wr.tensor(fields["running_mean"])), ("eps", lambda: wr.number(fields["eps"])),
                 ("train", lambda: wr.boolean(train))]
        items.append(("running_std" if old else "running_var", lambda: wr.tensor(fields["running_var"])))
        if fields.get("weight") is not None:
            items += [("weight", lambda: wr.tensor(fields["weight"])), ("bias", lambda: wr.tensor(fields["bias"]))]
        return lambda: wr.obj(cls, items)

    def node(i):
        if i in written:
            wr.i32(4)
            wr.i32(written[i])
            return
        cls, fields, name, children = nodes[i]
        if fields is None:
            mod = lambda: wr.obj(cls, [("train", lambda: wr.boolean(True))])
        elif isinstance(fields[0], str):
            mod = bn_mod(cls, *fields[1:])
        else:
            mod = conv(*fields)
        data = [("module", mod)]
        if name:
            data.append(("annotations", lambda: wr.table([("name", lambda: wr.string(name))])))
        wr.i32(4)
        written[i] = wr.next
        wr.i32(wr.next)
        wr.next += 1
        wr.s("V 1")
        wr.s("nngraph.Node")
        wr.table([("data", lambda: wr.table(data)),
                  ("children", lambda: wr.table([(k + 1, (lambda c=c: node(c))) for k, c in enumerate(children)]))])

    wr.obj("nn.gModule", [("forwardnodes", lambda: wr.table([(i + 1, (lambda i=i: node(i))) for i in range(len(nodes))]))])
    path.write_bytes(bytes(wr.b))


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


def mconf_for(is3d, bk, affine, **kw):
    extra = {"batchNormEps": 1e-4}
    if bk:
        extra.update({"banksNum": bk["num"], "banksSplitStage": bk["split_stage"], "banksJoinStage": bk["join_stage"],
                      "banksAggregateMethod": bk["aggregate"], "banksType": bk.get("type", "mres")})
    extra.update(kw)
    return mconf_of(is3d, addBatchNorm=True, batchNormAffine=affine, **extra)


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
