"""The reference's answers for exactly the inputs the tests give it.

Where oracle/_ref is built (BLITZAR_REFERENCE set at build time) the tests call the reference live.
Elsewhere they replay what the reference answered, recorded in tests/golden/reference_calls.npz and
keyed by a digest of the call's name and arguments, so a call whose inputs were never recorded fails
instead of passing. A live run with BLITZAR_RECORD_REFERENCE=<file.npz> writes the recorded calls
plus every call of that run to <file.npz>.
"""
import hashlib
import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_calls.npz")
# the pure entry points of oracle/refcpu.py and oracle/refgpu.py the tests use
CALLS = {"commit", "normalize", "random_elements", "ristretto_generators", "fixed_msm",
         "transcript_new", "transcript_challenge", "prove_inner_product", "verify_inner_product",
         "bucket_msm"}


def _feed(h, x):
    if isinstance(x, np.ndarray):
        a = np.ascontiguousarray(x)
        h.update(f"a{a.dtype.str}{a.shape}".encode())
        h.update(a.tobytes())
    elif isinstance(x, (list, tuple)):
        h.update(f"s{len(x)}(".encode())
        for y in x:
            _feed(h, y)
        h.update(b")")
    elif isinstance(x, (bytes, bytearray)):
        h.update(b"b%d:" % len(x) + bytes(x))
    elif isinstance(x, (bool, np.bool_)):
        h.update(b"T" if x else b"F")
    elif isinstance(x, (int, np.integer)):
        h.update(b"i%d;" % int(x))
    elif x is None:
        h.update(b"N")
    else:
        raise TypeError(f"unsupported argument type {type(x)}")


def digest(module, name, args, kwargs):
    h = hashlib.sha256(f"{module}.{name}".encode())
    _feed(h, list(args))
    for k in sorted(kwargs):
        h.update(k.encode())
        _feed(h, kwargs[k])
    return h.hexdigest()[:32]


class RecordedReference:
    """Stands in for oracle.refcpu / oracle.refgpu: live when `module` is given, replayed otherwise."""

    def __init__(self, label, module=None, store=None):
        self.label, self._m, self.live = label, module, module is not None
        self._store = store

    def available(self):
        return True

    def __getattr__(self, name):
        if name not in CALLS:
            raise AttributeError(name)
        return lambda *a, **kw: self._call(name, a, kw)

    def _call(self, name, args, kwargs):
        key = digest(self.label, name, args, kwargs)
        if self.live:
            before = {i: a.copy() for i, a in enumerate(args) if isinstance(a, np.ndarray)}
            res = getattr(self._m, name)(*args, **kwargs)
            changed = {i: args[i].copy() for i, b in before.items() if not np.array_equal(b, args[i])}
            self._store.put(key, res, changed)
            return res
        res, changed = self._store.get(key, f"{self.label}.{name}")
        for i, v in changed.items():
            args[i][...] = v
        return res


class Store:
    def __init__(self, path=GOLDEN):
        self.data = dict(np.load(path)) if os.path.exists(path) else {}
        self.new = {}

    def put(self, key, res, changed):
        items = list(res) if isinstance(res, tuple) else [res]
        self.new[key + ".t"] = np.array(isinstance(res, tuple))
        for j, r in enumerate(items):
            self.new[f"{key}.{j}"] = np.array(r)  # a copy: callers may advance a result in place
        for i, v in changed.items():
            self.new[f"{key}.m{i}"] = v

    def get(self, key, what):
        if key + ".t" not in self.data:
            raise AssertionError(f"{what}: no recorded reference answer for these inputs "
                                 f"({os.path.relpath(GOLDEN)}); build oracle/_ref to run it live")
        items, changed, j = [], {}, 0
        while f"{key}.{j}" in self.data:
            v = self.data[f"{key}.{j}"]
            items.append(v.item() if v.ndim == 0 else v.copy())
            j += 1
        for k, v in self.data.items():
            if k.startswith(key + ".m"):
                changed[int(k[len(key) + 2:])] = v
        return (tuple(items) if self.data[key + ".t"] else items[0]), changed

    def save(self, path):
        merged = dict(self.data)
        merged.update(self.new)
        np.savez_compressed(path, **merged)
