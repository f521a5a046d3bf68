"""The compiled reference's answers, recorded for machines without the reference sources.

oracle/_ref (the reference's own CPU code, compiled in place) exists only where the reference tree does.
Elsewhere the tests that pin the oracle on it get a ReplayReference: the same method surface, answering
from tests/golden/ref_calls.json.gz, which holds, per call (keyed by the method name and the exact bytes
of every argument), what the compiled reference returned (or the error it raised) and what it left in the
arrays it writes in place.  Small outputs are stored whole; larger ones by a digest of their float32 bits, which is all a
bit-for-bit comparison (cases.bits_equal) needs.  A call whose inputs were never recorded fails.

Regenerate, where oracle/_ref is built:
    TFL_RECORD_REFERENCE=1 python -m pytest tests/test_oracle_*.py -p no:cacheprovider
"""
import atexit
import base64
import gzip
import hashlib
import json
import os

import numpy as np

PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_calls.json.gz")
FULL_MAX = 64            # outputs up to this many elements are stored whole
ALWAYS_FULL = {"emptyDomain", "findConnectedFluidComponents", "flagsToOccupancy", "normalizePressureMean",
               "velocityUpdateBackward"}


def call_key(name, args):
    h = hashlib.sha1(name.encode())
    for a in args:
        if isinstance(a, np.ndarray):
            a = np.ascontiguousarray(a)
            h.update(("%s%s" % (a.dtype.str, a.shape)).encode())
            h.update(a.tobytes())
        else:
            h.update(repr(a).encode())
        h.update(b"|")
    return h.hexdigest()[:20]


def digest(a):
    a = np.ascontiguousarray(a, np.float32)
    return hashlib.sha1(repr(a.shape).encode() + a.tobytes()).hexdigest()


class Recorded:
    """An output of the compiled reference known by shape and the digest of its float32 bits."""

    def __init__(self, shape, dig):
        self.shape, self.digest = tuple(shape), dig

    def matches(self, a):
        return tuple(np.shape(a)) == self.shape and digest(a) == self.digest


# arrays a replayed call would have written in place, by id (the array itself is kept alive with it)
_inplace = {}


def expected(x):
    """x, or the Recorded output the replayed reference left in it."""
    if isinstance(x, np.ndarray) and id(x) in _inplace and _inplace[id(x)][0] is x:
        return _inplace[id(x)][1]
    return x


def _encode(name, a):
    if isinstance(a, np.ndarray):
        a = np.ascontiguousarray(a)
        if a.size <= FULL_MAX or name in ALWAYS_FULL:
            return {"dtype": a.dtype.str, "shape": list(a.shape), "data": base64.b64encode(a.tobytes()).decode()}
        return {"shape": list(a.shape), "digest": digest(a)}
    if isinstance(a, tuple):
        return {"tuple": [_encode(name, v) for v in a]}
    if isinstance(a, (np.generic,)):
        a = a.item()
    return {"value": a}


def _decode(e):
    if "tuple" in e:
        return tuple(_decode(v) for v in e["tuple"])
    if "value" in e:
        return e["value"]
    if "digest" in e:
        return Recorded(e["shape"], e["digest"])
    return np.frombuffer(base64.b64decode(e["data"]), np.dtype(e["dtype"])).reshape(e["shape"]).copy()


class RecordingReference:
    """Wraps oracle.Reference and records every call (written to PATH when the process exits)."""
    _calls = {}

    def __init__(self, real):
        self._real = real
        self.name = real.name
        if not RecordingReference._calls:
            atexit.register(RecordingReference.save)

    def num_threads(self):
        return self._real.num_threads()

    def __getattr__(self, name):
        fn = getattr(self._real, name)

        def call(*args):
            key = call_key(name, args)
            before = [a.copy() if isinstance(a, np.ndarray) else None for a in args]
            try:
                out = fn(*args)
            except RuntimeError as e:
                RecordingReference._calls[key] = {"raises": str(e)}
                raise
            written = {str(i): _encode(name, a) for i, (a, b) in enumerate(zip(args, before))
                       if b is not None and not np.array_equal(a.view(np.uint8), b.view(np.uint8))}
            RecordingReference._calls[key] = {"out": _encode(name, out), "inplace": written}
            return out
        return call

    @staticmethod
    def save():
        with gzip.open(PATH, "wt") as f:
            json.dump(RecordingReference._calls, f, sort_keys=True, separators=(",", ":"))


class ReplayReference:
    name = "reference"
    _calls = None

    def __init__(self):
        if ReplayReference._calls is None:
            with gzip.open(PATH, "rt") as f:
                ReplayReference._calls = json.load(f)

    def num_threads(self):
        return 1

    def __getattr__(self, name):
        def call(*args):
            rec = ReplayReference._calls.get(call_key(name, args))
            assert rec is not None, "no recorded reference answer for this %s call (inputs changed?)" % name
            if "raises" in rec:
                raise RuntimeError(rec["raises"])
            for i, e in rec["inplace"].items():
                v = _decode(e)
                if isinstance(v, Recorded):
                    _inplace[id(args[int(i)])] = (args[int(i)], v)
                else:
                    np.copyto(args[int(i)], v)
            return _decode(rec["out"])
        return call


def reference():
    """The compiled reference where it is built (recording when TFL_RECORD_REFERENCE is set), else its replay."""
    import oracle
    if oracle.have_reference():
        real = oracle.Reference()
        return RecordingReference(real) if os.environ.get("TFL_RECORD_REFERENCE") else real
    return ReplayReference()
