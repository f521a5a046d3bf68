"""Writers of the reference's Torch7 files for the tests: the binary serializer, the nngraph networks of the plain,
banked, batch-normalized and dilated graphs, and their _mconf.bin tables."""
import os
import struct

import numpy as np


GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "myModel2D_layers.npz")


REF_MODEL = "/root/reference/data/models/myModel2D"


class W:
    """Minimal Torch7 binary writer (torch7/File.lua conventions)."""

    def __init__(self):
        self.b = bytearray()
        self.next = 1

    def i32(self, v): self.b += struct.pack("<i", v)
    def i64(self, v): self.b += struct.pack("<q", v)
    def s(self, v): self.i32(len(v)); self.b += v.encode()

    def number(self, v): self.i32(1); self.b += struct.pack("<d", v)
    def string(self, v): self.i32(2); self.s(v)
    def boolean(self, v): self.i32(5); self.i32(1 if v else 0)

    def table(self, items):
        self.i32(3); self.i32(self.next); self.next += 1
        self.i32(len(items))
        for k, wv in items:
            (self.number if not isinstance(k, str) else self.string)(k)
            wv()

    def backref_table(self, idx): self.i32(3); self.i32(idx)

    def tensor(self, a, cls="torch.FloatTensor", storage_cls="torch.FloatStorage"):
        a = np.ascontiguousarray(a, np.float32)
        self.i32(4); self.i32(self.next); self.next += 1
        self.s("V 1"); self.s(cls)
        self.i32(a.ndim)
        for d in a.shape: self.i64(d)
        stride = [int(np.prod(a.shape[i + 1:])) for i in range(a.ndim)]
        for d in stride: self.i64(d)
        self.i64(1)
        self.i32(4); self.i32(self.next); self.next += 1
        self.s("V 1"); self.s(storage_cls)
        self.i64(a.size); self.b += a.tobytes()

    def obj(self, cls, items):
        self.i32(4); self.i32(self.next); self.next += 1
        self.s("V 1"); self.s(cls)
        self.table(items)


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


def mconf_for(is3d, bk, affine, **kw):
    extra = {"batchNormEps": 1e-4}
    if bk:
        extra.update({"banksNum": bk["num"], "banksSplitStage": bk["split_stage"], "banksJoinStage": bk["join_stage"],
                      "banksAggregateMethod": bk["aggregate"], "banksType": bk.get("type", "mres")})
    extra.update(kw)
    return mconf_of(is3d, addBatchNorm=True, batchNormAffine=affine, **extra)


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


def write_mconf(path, mconf):
    wr = W()

    def value(v):
        if isinstance(v, bool):
            return lambda: wr.boolean(v)
        if isinstance(v, (int, float)):
            return lambda: wr.number(v)
        if isinstance(v, str):
            return lambda: wr.string(v)
        return lambda: wr.table([(k, value(x)) for k, x in v.items()])

    value(mconf)()
    path.write_bytes(bytes(wr.b))
