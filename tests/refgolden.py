"""Differential checks against the unmodified reference that also run where it is not built.

`check(name, port_value, ref_call)` compares what the oracle computed with what the reference
computes.  Where oracle/_ref/libref.so is built, ref_call() runs and the two must be equal; where
it is not, the oracle's value must have the SHA-256 the reference's value had when
tests/golden/ref_digests.json was recorded (RSB200_RECORD_GOLDEN=1 with the reference built
rewrites that file from the reference's own results)."""
import hashlib
import json
import os

import numpy as np

import oracle
from oracle import port

PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_digests.json")
RECORD = os.environ.get("RSB200_RECORD_GOLDEN") == "1"
_golden = json.load(open(PATH)) if os.path.exists(PATH) else {}


def outcome(fn):
    """fn()'s value, or the class of the oracle error it raised."""
    try:
        return fn()
    except port.OracleError as e:
        return ("raises", type(e).__name__)


def digest(v):
    h = hashlib.sha256()

    def feed(x):
        if isinstance(x, np.ndarray):
            h.update(("nd%s%s" % (x.dtype.str, x.shape)).encode())
            h.update(np.ascontiguousarray(x).tobytes())
        elif isinstance(x, (bytes, bytearray)):
            h.update(b"by%d:" % len(x) + bytes(x))
        elif isinstance(x, (list, tuple)):
            h.update(b"[%d" % len(x))
            for y in x:
                feed(y)
            h.update(b"]")
        elif isinstance(x, (bool, np.bool_)):
            h.update(b"b1" if x else b"b0")
        elif isinstance(x, (int, np.integer)):
            h.update(b"i%d;" % int(x))
        elif isinstance(x, str):
            h.update(b"s" + x.encode() + b";")
        else:
            raise TypeError(type(x))
    feed(v)
    return h.hexdigest()[:16]


def _equal(a, b):
    if isinstance(a, np.ndarray) or isinstance(b, np.ndarray):
        return isinstance(a, np.ndarray) and isinstance(b, np.ndarray) and np.array_equal(a, b)
    if isinstance(a, (list, tuple)) and isinstance(b, (list, tuple)):
        return len(a) == len(b) and all(_equal(x, y) for x, y in zip(a, b))
    return a == b


def check(name, port_value, ref_call):
    if oracle.HAVE_REF:
        want = ref_call()
        if RECORD:
            _golden[name] = digest(want)
            with open(PATH, "w") as f:
                json.dump(_golden, f, indent=0, sort_keys=True)
        assert _equal(port_value, want), name
    else:
        assert name in _golden, "no recorded reference result for %s" % name
        assert digest(port_value) == _golden[name], name
