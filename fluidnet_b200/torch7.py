"""Reader for Torch7's binary serialization (torch.save / torch.DiskFile():binary()) -- enough of it to
bring a model trained with the reference into this library without Torch7: the network file written by
torch/lib/save_model.lua and the `_mconf.bin` table beside it (torch/lib/load_model.lua).

Format (torch7/File.lua, the un-vendored Torch7 distro the reference runs on): every value starts with an
int32 type tag -- 0 nil, 1 number (float64), 2 string (int32 length + bytes), 3 table, 4 torch object,
5 boolean, 6/7/8 functions.  Tables and torch objects carry an int32 index first; an index seen before is
a back-reference.  A torch object continues with a version string ("V 1"), its class name and the class's
own payload: tensors write ndim, sizes, strides (int64 each), storage offset (1-based) and their storage
object; storages write their length and the raw elements; every other class (nn modules, nngraph nodes)
writes one table with its fields.  torch.Cuda* tensors / storages are written like their Float versions.
Host-side only, no GPU involved.
"""
import re
import struct

import numpy as np

_STORAGE_DTYPES = {
    "torch.FloatStorage": np.float32, "torch.CudaStorage": np.float32, "torch.DoubleStorage": np.float64,
    "torch.CudaDoubleStorage": np.float64, "torch.LongStorage": np.int64, "torch.CudaLongStorage": np.int64,
    "torch.IntStorage": np.int32, "torch.CudaIntStorage": np.int32, "torch.ByteStorage": np.uint8,
    "torch.CudaByteStorage": np.uint8, "torch.CharStorage": np.int8, "torch.ShortStorage": np.int16,
    "torch.HalfStorage": np.float16, "torch.CudaHalfStorage": np.float16,
}


class T7Object:
    """A torch class instance that is not a tensor / storage: `cls` and its field table `fields`."""

    def __init__(self, cls, fields):
        self.cls = cls
        self.fields = fields

    def __getitem__(self, key):
        return self.fields[key]

    def get(self, key, default=None):
        return self.fields.get(key, default) if isinstance(self.fields, dict) else default

    def __repr__(self):
        return "T7Object(%s)" % self.cls


class _ObjKey:
    """A table / object used as a table key (nngraph keeps node -> node maps): hashable by identity."""

    def __init__(self, obj):
        self.obj = obj

    def __hash__(self):
        return id(self.obj)

    def __eq__(self, other):
        return isinstance(other, _ObjKey) and other.obj is self.obj


class _Reader:
    def __init__(self, data):
        self.d = data
        self.o = 0
        self.memo = {}

    def _unpack(self, fmt, size):
        v = struct.unpack_from(fmt, self.d, self.o)
        self.o += size
        return v[0]

    def int32(self):
        return self._unpack("<i", 4)

    def int64(self):
        return self._unpack("<q", 8)

    def float64(self):
        return self._unpack("<d", 8)

    def string(self):
        n = self.int32()
        s = self.d[self.o:self.o + n].decode("latin-1")
        self.o += n
        return s

    def value(self):
        tag = self.int32()
        if tag == 0:
            return None
        if tag == 1:
            v = self.float64()
            return int(v) if (v == v and abs(v) < 2 ** 53 and v == int(v)) else v
        if tag == 2:
            return self.string()
        if tag == 5:
            return self.int32() == 1
        if tag == 3:
            idx = self.int32()
            if idx in self.memo:
                return self.memo[idx]
            t = {}
            self.memo[idx] = t
            n = self.int32()
            for _ in range(n):
                k = self.value()
                if isinstance(k, (dict, T7Object, np.ndarray)):
                    k = _ObjKey(k)
                t[k] = self.value()
            return t
        if tag == 4:
            idx = self.int32()
            if idx in self.memo:
                return self.memo[idx]
            version = self.string()
            cls = self.string() if version.startswith("V ") else version
            return self._torch_object(idx, cls)
        if tag in (6, 7, 8):                     # functions: dumped bytecode (+ upvalues); skipped
            if tag in (7, 8):
                idx = self.int32()
                if idx in self.memo:
                    return self.memo[idx]
                self.memo[idx] = "<function>"
            self.string()                        # the dump
            if tag in (7, 8):
                self.value()                     # upvalues table
            return "<function>"
        raise ValueError("torch7 file: unknown type tag %d at offset %d" % (tag, self.o - 4))

    def _torch_object(self, idx, cls):
        if cls in _STORAGE_DTYPES:
            n = self.int64()
            dt = np.dtype(_STORAGE_DTYPES[cls])
            a = np.frombuffer(self.d, dtype=dt, count=n, offset=self.o).copy()
            self.o += n * dt.itemsize
            self.memo[idx] = a
            return a
        if cls.endswith("Tensor") and cls.startswith("torch."):
            nd = self.int32()
            size = [self.int64() for _ in range(nd)]
            stride = [self.int64() for _ in range(nd)]
            offset = self.int64() - 1
            storage = self.value()
            if storage is None or nd == 0:
                a = np.zeros(size if nd else (0,), np.float32)
            else:
                a = np.lib.stride_tricks.as_strided(storage[offset:], shape=size,
                                                    strides=[s * storage.itemsize for s in stride]).copy()
            self.memo[idx] = a
            return a
        obj = T7Object(cls, None)
        self.memo[idx] = obj
        obj.fields = self.value()
        return obj


def load(path):
    """Deserialize the first value of a Torch7 binary file."""
    import sys
    with open(path, "rb") as f:
        data = f.read()
    limit = sys.getrecursionlimit()
    sys.setrecursionlimit(max(limit, 20000))         # nngraph models nest deeply (node -> children -> node ...)
    try:
        return _Reader(data).value()
    finally:
        sys.setrecursionlimit(limit)


def _walk(obj, seen, out):
    """Depth-first over tables / objects in insertion order, collecting convolution modules."""
    if id(obj) in seen:
        return
    if isinstance(obj, T7Object):
        seen.add(id(obj))
        if obj.cls.endswith("Convolution") and isinstance(obj.fields, dict) and "weight" in obj.fields:
            out.append(obj)
            return
        _walk(obj.fields, seen, out)
    elif isinstance(obj, dict):
        seen.add(id(obj))
        keys = list(obj.keys())
        ints = sorted(k for k in keys if isinstance(k, int))
        for k in ints + [k for k in keys if not isinstance(k, int)]:
            if isinstance(k, _ObjKey):
                _walk(k.obj, seen, out)
            _walk(obj[k], seen, out)


def conv_layers(model):
    """[(weight [cout][cin][kz][ky][kx], bias [cout]), ...] of a deserialized reference model, in forward
    order.  The reference's graphs are nngraph gModules: `forwardnodes` is already topologically sorted
    (nngraph/gmodule.lua), so the convolutions are taken from there; a plain nn.Sequential is walked in
    module order."""
    convs = []
    nodes = model.get("forwardnodes") if isinstance(model, T7Object) else None
    if nodes:
        for i in sorted(nodes):
            data = nodes[i].get("data") if isinstance(nodes[i], T7Object) else None
            mod = data.get("module") if isinstance(data, dict) else None
            if mod is not None:
                _walk(mod, set(), convs)
    else:
        _walk(model, set(), convs)
    return _conv_layers_of(convs)


def _conv_layers_of(convs):
    layers = []
    for c in convs:
        w = np.asarray(c["weight"], np.float32)
        b = np.asarray(c["bias"], np.float32).reshape(-1)
        cout, cin = int(c["nOutputPlane"]), int(c["nInputPlane"])
        if "kT" in c.fields:                                     # Volumetric: kT x kH x kW
            k = (int(c["kT"]), int(c["kH"]), int(c["kW"]))
        else:                                                    # Spatial: kH x kW
            k = (1, int(c["kH"]), int(c["kW"]))
        layers.append((np.ascontiguousarray(w.reshape(cout, cin, *k)), np.ascontiguousarray(b)))
    return layers


_CONV_STAGE = re.compile(r"^Bank (\d+): conv stage (\d+)$")

# Node modules of the graphs this library computes (lib/model.lua:27-401 with the options model_options accepts).
_ALLOWED = {
    "nn.Identity", "nn.SelectTable", "nn.Select", "nn.Unsqueeze", "nn.JoinTable", "nn.CAddTable", "nn.ApplyScale",
    "nn.Sequential", "tfluids.SetWallBcs", "tfluids.VelocityDivergence", "tfluids.FlagsToOccupancy",
    "tfluids.VelocityUpdate", "tfluids.VolumetricUpSamplingNearest", "nn.SpatialUpSamplingNearest",
    "nn.ReLU", "cudnn.ReLU", "nn.Sigmoid", "cudnn.Sigmoid", "nn.ReLU6",
    "nn.SpatialConvolution", "nn.VolumetricConvolution", "cudnn.SpatialConvolution", "cudnn.VolumetricConvolution",
    "nn.SpatialConvolutionUpsample", "nn.VolumetricConvolutionUpsample",
    "nn.SpatialAveragePooling", "nn.VolumetricAveragePooling", "cudnn.SpatialAveragePooling",
    "cudnn.VolumetricAveragePooling", "nn.SpatialMaxPooling", "nn.VolumetricMaxPooling", "cudnn.SpatialMaxPooling",
    "cudnn.VolumetricMaxPooling",
}

# The convolutions of banks 2..N of a banksType 'dilate' model (lib/model_utils.lua:122-146).
_DILATED = {"nn.SpatialDilatedConvolution", "nn.VolumetricDilatedConvolution"}

# torch.addBN (lib/model_utils.lua:36-62): cudnn.* with batchNormAffine, nn.* (no weight / bias) without.
_BATCH_NORM = {"nn.SpatialBatchNormalization", "nn.VolumetricBatchNormalization", "cudnn.SpatialBatchNormalization",
               "cudnn.VolumetricBatchNormalization"}
# The nodes between a stage's convolution and its batch normalization (lib/model.lua:337-350).
_NONLIN_POOL = {"nn.ReLU", "cudnn.ReLU", "nn.Sigmoid", "cudnn.Sigmoid", "nn.ReLU6",
                "nn.SpatialAveragePooling", "nn.VolumetricAveragePooling", "cudnn.SpatialAveragePooling",
                "cudnn.VolumetricAveragePooling", "nn.SpatialMaxPooling", "nn.VolumetricMaxPooling",
                "cudnn.SpatialMaxPooling", "cudnn.VolumetricMaxPooling"}


def _check_dilation(conv, cls, bank):
    """banksType 'dilate' (lib/model.lua:319-322, lib/model_utils.lua:122-146): the convolution of bank i >= 2 is an
    nn.{Spatial,Volumetric}DilatedConvolution with dilation 2^(i-1) on every axis, stride 1 and padding
    2^(i-1) (k-1)/2; bank 1's convolutions and the ones outside the banks are ordinary ones."""
    where = "bank %d's convolution" % bank if bank else "the final convolution"
    if cls not in _DILATED:
        if bank and bank > 1:
            raise ValueError("torch7 model: %s of a banksType 'dilate' model is %s, not a dilated convolution"
                             % (where, cls))
        return
    if not bank or bank == 1:
        raise ValueError("torch7 model: %s is %s; only banks 2.. of a banksType 'dilate' model are dilated"
                         % (where, cls))
    d = 2 ** (bank - 1)
    for a in (("T", "W", "H") if cls == "nn.VolumetricDilatedConvolution" else ("W", "H")):
        k = int(conv["k" + a])
        got = tuple(None if conv.get(f) is None else int(conv.get(f)) for f in ("dilation" + a, "pad" + a, "d" + a))
        want = (d, d * (k - 1) // 2, 1)
        if got != want:
            raise ValueError("torch7 model: %s (%s) has (dilation, pad, stride) %s = %s on axis %s; banksType "
                             "'dilate' gives %s" % (where, cls, "dilation%s, pad%s, d%s" % (a, a, a), got, a, want))


# (osize, ksize, psize, usize) per modelType, lib/model.lua:163-239.
_ARCH = {
    (False, "default"): ([16, 16, 16, 16, 1], [3, 3, 3, 3, 1], [1] * 5, [1] * 5),
    (False, "tog"): ([16, 32, 32, 64, 64, 32, 1], [5, 5, 5, 5, 1, 1, 3], [2, 1, 1, 1, 1, 1, 1], [1, 1, 1, 1, 1, 1, 2]),
    (False, "yang"): ([6, 6, 6, 1], [3, 1, 1, 1], [1] * 4, [1] * 4),
    (True, "default"): ([8, 8, 8, 8, 1], [3, 3, 3, 1, 1], [1] * 5, [1] * 5),
    (True, "tog"): ([16, 16, 16, 16, 32, 32, 1], [3, 3, 3, 3, 1, 1, 3], [2, 2, 1, 1, 1, 1, 1], [1, 1, 1, 1, 1, 2, 2]),
    (True, "yang"): ([6, 6, 6, 1], [3, 1, 1, 1], [1] * 4, [1] * 4),
}


def _node_modules(model):
    """(module, annotation name or None) of every node of an nngraph gModule, in forward order."""
    nodes = model.get("forwardnodes") if isinstance(model, T7Object) else None
    out = []
    for i in sorted(nodes or {}):
        data = nodes[i].get("data") if isinstance(nodes[i], T7Object) else None
        mod = data.get("module") if isinstance(data, dict) else None
        if mod is None:
            continue
        ann = data.get("annotations")
        out.append((mod, ann.get("name") if isinstance(ann, dict) else None))
    return out


def graph_stages(model, dilate=False, batchnorm=False):
    """The convolutions of a reference gModule grouped by stage: [[(weight, bias) of bank 1, bank 2, ...], ...].
    Each convolution is assigned from its node's annotation "Bank i: conv stage l" (lib/model.lua:337); the final
    convolution has none.  Raises ValueError, naming it, for a module outside the graphs the library computes
    (batch normalisation, gated convolutions, low-rank convolution Sequentials, ...).  Dilated convolutions are such a
    module unless dilate=True, which reads a banksType 'dilate' model: bank i >= 2's convolutions must then be dilated
    by 2^(i-1) (see _check_dilation) and all others undilated.  Batch normalization modules are accepted with
    batchnorm=True only (batch_norm_layers reads them)."""
    mods = _node_modules(model)
    if not mods:
        raise ValueError("torch7 model: not an nngraph gModule (no forwardnodes)")
    found = {}
    final = []
    for mod, name in mods:
        cls = mod.cls if isinstance(mod, T7Object) else type(mod).__name__
        if cls not in _ALLOWED and not (dilate and cls in _DILATED) and not (batchnorm and cls in _BATCH_NORM):
            raise ValueError("torch7 model: module %s is not supported by this library" % cls)
        convs = []
        _walk(mod, set(), convs)
        if cls == "nn.Sequential":
            if convs:
                raise ValueError("torch7 model: a convolution inside nn.Sequential (low-rank convolution) is not "
                                 "supported by this library")
            continue
        if not convs:
            continue
        layer = _conv_layers_of(convs)
        if len(layer) != 1:
            raise ValueError("torch7 model: module %s holds %d convolutions" % (cls, len(layer)))
        m = _CONV_STAGE.match(name or "")
        if dilate:
            _check_dilation(convs[0], cls, int(m.group(1)) if m else None)
        if m:
            key = (int(m.group(2)), int(m.group(1)))
            if key in found:
                raise ValueError("torch7 model: two convolutions annotated %r" % name)
            found[key] = layer[0]
        else:
            final.append(layer[0])
    if len(final) != 1:
        raise ValueError("torch7 model: expected one final (unannotated) convolution, found %d" % len(final))
    n_stages = max([s for s, _ in found] + [0]) + 1
    stages = []
    for s in range(1, n_stages):
        banks = sorted(b for st, b in found if st == s)
        if not banks:
            raise ValueError("torch7 model: no convolution is annotated with stage %d" % s)
        if banks != list(range(1, len(banks) + 1)):
            raise ValueError("torch7 model: stage %d has convolutions of banks %s" % (s, banks))
        convs = [found[(s, b)] for b in banks]
        stages.append(convs if len(convs) > 1 else convs[0])
    stages.append(final[0])
    return stages


def _cls(obj):
    return obj.cls if isinstance(obj, T7Object) else type(obj).__name__


def batch_norm_layers(model):
    """The batch normalization of an addBatchNorm gModule (lib/model.lua:343-350) as ProjectionModel's batchNorm:
    {"train": bool, "layers": [...]} with "layers" mirroring graph_stages(model)[:-1] (a list per banked stage, bank
    order), each entry {"weight", "bias" (None without affine parameters), "running_mean", "running_var", "eps",
    "cls"}.  BN nodes carry no annotation, so each is assigned to the convolution whose node reaches it through the
    graph's edges (`children`) across non-linearity and pooling nodes only.  Raises ValueError, naming it, for a BN
    module reached from no stage convolution, a stage convolution without one, a channel count other than the
    convolution's, modules whose `train` flags differ, and an old-format module (running_std without running_var)."""
    nodes = model.get("forwardnodes") if isinstance(model, T7Object) else None
    if not nodes:
        raise ValueError("torch7 model: not an nngraph gModule (no forwardnodes)")
    order = [nodes[i] for i in sorted(nodes) if isinstance(nodes[i], T7Object)]

    def data(node):
        d = node.get("data")
        return d if isinstance(d, dict) else {}

    def children(node):
        ch = node.get("children")
        return [ch[k] for k in sorted(k for k in ch if isinstance(k, int))] if isinstance(ch, dict) else []

    assigned = {}       # id(BN node) -> (stage, bank)
    stage_conv = {}     # (stage, bank) -> conv module
    for node in order:
        d = data(node)
        ann = d.get("annotations")
        m = _CONV_STAGE.match((ann.get("name") if isinstance(ann, dict) else None) or "")
        if not m or d.get("module") is None:
            continue
        key = (int(m.group(2)), int(m.group(1)))
        stage_conv[key] = d["module"]
        todo, seen = list(children(node)), set()
        while todo:
            nd = todo.pop()
            if id(nd) in seen:
                continue
            seen.add(id(nd))
            cls = _cls(data(nd).get("module"))
            if cls in _BATCH_NORM:
                if id(nd) in assigned and assigned[id(nd)] != key:
                    raise ValueError("torch7 model: a %s is reached from two stage convolutions" % cls)
                assigned[id(nd)] = key
            elif cls in _NONLIN_POOL:
                todo += children(nd)
    found = {}
    trains = set()
    for node in order:
        mod = data(node).get("module")
        cls = _cls(mod)
        if cls not in _BATCH_NORM:
            continue
        if id(node) not in assigned:
            raise ValueError("torch7 model: %s is not placed after a stage's convolution, non-linearity and pooling "
                             "(lib/model.lua:343-350)" % cls)
        key = assigned[id(node)]
        if key in found:
            raise ValueError("torch7 model: stage %d bank %d has two batch normalizations (%s)" % (key + (cls,)))
        if mod.get("running_var") is None:
            if mod.get("running_std") is not None:
                raise ValueError("torch7 model: %s carries running_std without running_var (an old nn format this "
                                 "library does not read)" % cls)
            raise ValueError("torch7 model: %s has no running_var" % cls)
        mean = np.asarray(mod["running_mean"], np.float32).reshape(-1)
        var = np.asarray(mod["running_var"], np.float32).reshape(-1)
        conv = stage_conv[key]
        c = conv.get("nOutputPlane") if isinstance(conv, T7Object) else None
        if c is not None and mean.shape[0] != int(c):
            raise ValueError("torch7 model: %s of stage %d bank %d has %d channels, its convolution %d"
                             % (cls, key[0], key[1], mean.shape[0], int(c)))
        w, b = mod.get("weight"), mod.get("bias")
        trains.add(bool(mod.get("train", True)))
        found[key] = {"weight": None if w is None else np.asarray(w, np.float32).reshape(-1),
                      "bias": None if b is None else np.asarray(b, np.float32).reshape(-1),
                      "running_mean": mean, "running_var": var, "eps": float(mod.get("eps", 1e-5)), "cls": cls}
    if len(trains) > 1:
        raise ValueError("torch7 model: the batch normalization modules differ in their train flag")
    layers = []
    for s in range(1, max([k[0] for k in stage_conv] + [0]) + 1):
        banks = sorted(b for st, b in stage_conv if st == s)
        missing = [b for b in banks if (s, b) not in found]
        if missing:
            raise ValueError("torch7 model: stage %d bank %d has no batch normalization" % (s, missing[0]))
        entries = [found[(s, b)] for b in banks]
        layers.append(entries if len(entries) > 1 else entries[0])
    return {"train": trains.pop() if trains else True, "layers": layers}


def input_options(mconf):
    """The input block of a reference mconf (lib/model.lua:27-150, :357-387; defaults lib/default_conf.lua:45-47,
    76-81, 103-106) as ProjectionModel keyword arguments.  Raises ValueError naming the key for every combination the
    reference cannot build, with the reference's own message where it has one."""
    def opt(key, default=None):
        return mconf.get(key, default)

    def bad(key, why):
        raise ValueError("mconf: %s: %s" % (key, why))

    chans = {"pDiv": False, "UDiv": False, "div": False, "flags": False}
    given = opt("inputChannels") or {"pDiv": True, "div": True, "flags": True}
    for k, v in given.items():
        if k not in chans:
            bad("inputChannels", "unknown channel %r" % k)
        chans[k] = bool(v)
    if not chans["flags"]:
        bad("inputChannels", "Are you sure you dont want flags on input?")                      # model.lua:39-43
    if not (chans["pDiv"] or chans["UDiv"] or chans["div"]):
        bad("inputChannels", "Are you sure you dont want any (U, div or p) fields?")            # :50-52
    if not (chans["UDiv"] or chans["div"]):
        bad("inputChannels", "tfluids.VelocityUpdate needs UDiv, which is selected only when UDiv or div is an "
                             "input (lib/model.lua:69-72, :380)")
    normalize = opt("normalizeInput", True)
    if normalize not in (True, False):
        bad("normalizeInput", "%r is not a boolean" % (normalize,))
    func = opt("normalizeInputFunc", "std")
    chan = opt("normalizeInputChan", "UDiv")
    if normalize:
        if func not in ("std", "norm"):
            bad("normalizeInputFunc", "Incorrect normalize input function (%r)" % (func,))       # :103
        if chan not in ("UDiv", "pDiv", "div"):
            bad("normalizeInputChan", "Incorrect normalize input channel. (%r)" % (chan,))       # :114
        if chan == "div" and not chans["div"]:
            bad("normalizeInputChan", "'div' needs inputChannels.div (lib/model.lua:108-116: div is nil)")
    else:
        func, chan = "std", "UDiv"      # unused without the scale node
    model_type = opt("modelType", "default")
    if model_type == "yang":                                                                     # model_utils.lua:211-227
        if not chans["pDiv"]:
            bad("inputChannels", "ERROR: yang model must have pDiv input")
        if not chans["div"]:
            bad("inputChannels", "ERROR: yang model must have div input")
        if chans["UDiv"]:
            bad("inputChannels", "ERROR: yang model must not have UDiv input")
    skip = bool(opt("addPressureSkip", False))
    if skip and model_type == "tog":
        bad("addPressureSkip", "'tog' joins pDiv to a half-resolution hidden layer before its upsampling last "
                               "convolution, which lib/model.lua:357-361 cannot build")
    return {"inputChannels": chans, "normalizeInput": bool(normalize), "normalizeInputFunc": func,
            "normalizeInputChan": chan, "addPressureSkip": skip}


def model_options(mconf, n_stages=None, inputs=False, dilate=False, batchnorm=False, relu6=False, bn=None):
    """ProjectionModel keyword arguments for a reference mconf (lib/default_conf.lua, lib/model.lua:27-401):
    pool / up from modelType, poolType, nonlinType, banks, normalizeInputThreshold, and with inputs=True the input
    block (input_options).  Raises ValueError, naming the option, for anything the library does not compute.  Without
    inputs=True a non-default input block is refused too: a caller that drops those keys would build another model.
    Likewise banksType 'dilate' is accepted with dilate=True only (banks["type"] = 'dilate'; the file's convolutions
    then come from graph_stages(model, dilate=True)), addBatchNorm with batchnorm=True only and nonlinType 'relu6'
    with relu6=True only.  bn (batch_norm_layers of the file) is checked against batchNormAffine (modules with or
    without weight and bias), batchNormEps and the channel count osize of each stage, and returned as "batchNorm"."""
    def opt(key, default=None):
        return mconf.get(key, default)

    def refuse(what):
        raise ValueError("mconf: %s is not supported by this library" % what)

    if opt("addBatchNorm") and not batchnorm:
        refuse("addBatchNorm = true (model_options(mconf, batchnorm=True) builds it)")
    if not inputs:
        if opt("addPressureSkip"):
            refuse("addPressureSkip = true (model_options(mconf, inputs=True) builds it)")
        chans = opt("inputChannels") or {"pDiv": True, "div": True, "flags": True}
        on = sorted(k for k, v in chans.items() if v)
        if on != ["div", "flags", "pDiv"]:
            refuse("inputChannels = {%s} (only pDiv, div, flags; model_options(mconf, inputs=True) builds the others)"
                   % ", ".join(on))
        if opt("normalizeInput", True) is not True:
            refuse("normalizeInput = false (model_options(mconf, inputs=True) builds it)")
        if opt("normalizeInputFunc", "std") != "std":
            refuse("normalizeInputFunc = %r (model_options(mconf, inputs=True) builds 'norm')" % opt("normalizeInputFunc"))
        if opt("normalizeInputChan", "UDiv") != "UDiv":
            refuse("normalizeInputChan = %r (model_options(mconf, inputs=True) builds 'pDiv', 'div')"
                   % opt("normalizeInputChan"))
    nonlin = opt("nonlinType", "relu")
    if nonlin == "relu6" and not relu6:
        refuse("nonlinType = 'relu6' (model_options(mconf, relu6=True) builds it)")
    if nonlin not in ("relu", "sigmoid", "relu6"):
        refuse("nonlinType = %r" % nonlin)
    pool_type = opt("poolType", "avg")
    if pool_type not in ("avg", "max"):
        refuse("poolType = %r" % pool_type)
    key = (bool(opt("is3D")), opt("modelType", "default"))
    if key not in _ARCH:
        refuse("modelType = %r" % key[1])
    _, _, psize, usize = _ARCH[key]
    out = {"pool": list(psize), "up": list(usize), "poolType": pool_type, "nonlinType": nonlin,
           "normalizeInputThreshold": float(opt("normalizeInputThreshold", 1e-5))}
    num = int(opt("banksNum", 1))
    if num > 1:
        btype = opt("banksType", "mres")
        if btype == "dilate" and not dilate:
            refuse("banksType = 'dilate' (model_options(mconf, dilate=True) builds it)")
        if btype not in ("mres", "dilate"):
            refuse("banksType = %r" % btype)
        if opt("banksWeightShare"):
            refuse("banksWeightShare = true")
        agg = opt("banksAggregateMethod", "concat")
        if agg not in ("concat", "add"):
            refuse("banksAggregateMethod = %r" % agg)
        out["banks"] = {"num": num, "split_stage": int(opt("banksSplitStage", 1)),
                        "join_stage": int(opt("banksJoinStage", 3)), "aggregate": agg}
        if btype == "dilate":
            out["banks"]["type"] = "dilate"
            s, j = out["banks"]["split_stage"], out["banks"]["join_stage"]
            if any(u > 1 for u in usize[s - 1:j - 1]):                                  # model_utils.lua:125
                raise ValueError("mconf: banksType = 'dilate': upsampling not supported for dilated convolutions.")
    if inputs:
        out.update(input_options(mconf))
    if opt("addBatchNorm"):
        if bn is None:
            raise ValueError("mconf: addBatchNorm = true needs the file's batch normalization (bn=batch_norm_layers)")
        _check_batch_norm(bn, mconf, _ARCH[key][0])
        out["batchNorm"] = {"train": bn["train"], "layers": bn["layers"]}
    return out


def _check_batch_norm(bn, mconf, osize):
    """batchNormAffine (default true), batchNormEps (default 1e-4) and osize against the modules (model_utils.lua:36-62)."""
    affine = bool(mconf.get("batchNormAffine", True))
    eps = float(mconf.get("batchNormEps", 1e-4))
    if len(bn["layers"]) != len(osize) - 1:
        raise ValueError("torch7 model: batch normalization in %d stages, the mconf gives %d"
                         % (len(bn["layers"]), len(osize) - 1))
    for s, layer in enumerate(bn["layers"], start=1):
        for e in (layer if isinstance(layer, list) else [layer]):
            if (e["weight"] is not None) != affine or e["cls"].startswith("cudnn.") != affine:
                raise ValueError("mconf: batchNormAffine = %s, but stage %d holds %s %s weight and bias"
                                 % (str(affine).lower(), s, e["cls"], "with" if e["weight"] is not None else "without"))
            if e["eps"] != eps:
                raise ValueError("mconf: batchNormEps = %g, but stage %d's %s has eps %g" % (eps, s, e["cls"], e["eps"]))
            if e["running_mean"].shape[0] != osize[s - 1]:
                raise ValueError("torch7 model: stage %d's batch normalization has %d channels, osize is %d"
                                 % (s, e["running_mean"].shape[0], osize[s - 1]))


def check_stages(stages, mconf, options):
    """The file's convolutions against the architecture the mconf describes (lib/model.lua:163-361), the first taking
    the mconf's input channels and the last one more with addPressureSkip."""
    is3d = bool(mconf.get("is3D"))
    osize, ksize, _, usize = _ARCH[(is3d, mconf.get("modelType", "default"))]
    if len(stages) != len(osize):
        raise ValueError("torch7 model: %d stages, modelType %r has %d" % (len(stages), mconf.get("modelType"), len(osize)))
    bk = options.get("banks")
    ins = input_options(mconf)
    ch = ins["inputChannels"]
    cin = int(ch["pDiv"]) + (3 if is3d else 2) * int(ch["UDiv"]) + int(ch["div"]) + int(ch["flags"])
    for s, layer in enumerate(stages, start=1):
        convs = layer if isinstance(layer, list) else [layer]
        banked = bk is not None and bk["split_stage"] <= s < bk["join_stage"]
        if len(convs) != (bk["num"] if banked else 1):
            raise ValueError("torch7 model: stage %d has %d banks, the mconf gives %d" %
                             (s, len(convs), bk["num"] if banked else 1))
        if bk is not None and s == bk["join_stage"] and bk["aggregate"] == "concat":
            cin *= bk["num"]
        if s == len(osize) and ins["addPressureSkip"]:
            cin += 1                    # lib/model.lua:357-361: [hidden, pDiv]
        want = (osize[s - 1] * usize[s - 1] ** (3 if is3d else 2), cin, ksize[s - 1])
        for w, _ in convs:
            if (w.shape[0], w.shape[1], w.shape[4]) != want:
                raise ValueError("torch7 model: stage %d convolution is (cout, cin, k) = %s, the mconf gives %s" %
                                 (s, (w.shape[0], w.shape[1], w.shape[4]), want))
        cin = osize[s - 1]


def load_reference_model(model_path, mconf_path=None):
    """The pieces fluidnet_b200.model.ProjectionModel needs from a model saved by the reference
    (torch/lib/save_model.lua): {'is3D', 'layers', 'mconf'}.  `mconf_path` defaults to
    `<model_path>_mconf.bin` (torch/lib/load_model.lua)."""
    mconf = load(mconf_path or (model_path + "_mconf.bin"))
    model = load(model_path)
    if isinstance(model, dict) and "model" in model:
        model = model["model"]
    return {"is3D": bool(mconf.get("is3D")), "layers": conv_layers(model), "mconf": mconf, "model": model}
