"""Recorded answers of the unmodified reference solver, replayed in the tests that compare with it.

The reference CPU-indirect build (oracle/_ref/, compiled from the cvxgrp/scs sources by oracle/Makefile) exists only
where those sources do. The tests call it through `Reference`, which stands in for the ctypes library:

  * SCS_RECORD_REFERENCE=<dir> and the build present: every call goes to the real library, and what it returned --
    the return value, every double array it changed, ScsInfo / ScsSettings -- is recorded per test into <dir>/<test module>.npz;
  * otherwise the calls are answered from tests/golden/reference/<test module>.npz, in the order the test makes them.
    A module's record is one JSON index (key -> offset, length, dtype) over two flat blobs, float64 and uint8.

An array of at most FULL entries (or any array, for a Reference made with whole=True) is stored whole. A longer one is stored as a fixed sample: SAMPLE entries drawn
with a seed derived from its length, plus its entry of largest magnitude; on replay the other entries read NaN. Tests
therefore compare with the NaN-aware `rel` / `amax` below: the error is the largest one over the stored entries and the
scale (the largest magnitude) is exact.
"""
import ctypes as C
import json
import os
import weakref

import numpy as np

from scs_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN_DIR = os.path.join(ROOT, "tests", "golden", "reference")
REF_DIR = os.path.join(ROOT, "oracle", "_ref")
BUILDS = {"ref": "libscsindir_ref.so", "nolapack": "libscsindir_ref_nolapack.so", "omp": "libscsindir_ref_omp.so"}
FULL = 128
SAMPLE = 24

# data address -> the numpy array handed to C there through capi.dptr (ScsSolution holds bare pointers)
_arrays = weakref.WeakValueDictionary()
_dptr = capi.dptr


def _tracking_dptr(a):
    if a is not None:
        _arrays[a.ctypes.data] = a
    return _dptr(a)


capi.dptr = _tracking_dptr


def amax(v):
    """largest magnitude over the entries that are known (NaN = not stored)"""
    return float(np.nanmax(np.abs(v)))


def rel(a, b, floor=1.0):
    """max |a - b| / max(floor, max |b|) over the entries of b that are known; fails if none are"""
    assert not np.isnan(b).all(), "no stored reference entries to compare"
    return float(np.nanmax(np.abs(np.asarray(a) - np.asarray(b))) / max(floor, amax(b)))


def sample_index(size, peak):
    idx = np.random.default_rng(size).choice(size, SAMPLE, replace=False)
    return np.unique(np.append(idx, peak))


def _pack(v, whole):
    if whole or v.size <= FULL:
        return {"": v.copy()}
    a = np.abs(v)
    peak = int(np.argmax(np.where(np.isnan(a), -1.0, a)))
    return {"": v[sample_index(v.size, peak)], "#peak": np.array(peak)}


def _unpack(store, key, out):
    v = store[key]
    if key + "#peak" not in store:
        out[...] = v
        return
    out[...] = np.nan
    out[sample_index(out.size, int(store[key + "#peak"]))] = v


def _address(p):
    return C.cast(p, C.c_void_p).value


def _slots(args):
    """(slot name, numpy array) for every double array a call can write: pointer arguments and ScsSolution fields"""
    out = []
    for j, a in enumerate(args):
        if isinstance(a, C._Pointer) and a._type_ is C.c_double:
            arr = _arrays.get(_address(a)) if a else None
            if arr is not None:
                out.append((f"a{j}", arr))
        elif type(a).__name__ == "CArgObject" and isinstance(a._obj, capi.ScsSolution):
            for f in ("x", "y", "s"):
                p = getattr(a._obj, f)
                arr = _arrays.get(_address(p)) if p else None
                if arr is not None:
                    out.append((f"a{j}.{f}", arr))
    return out


def _infos(args):
    """structs a call fills in: ScsInfo, and ScsSettings (scs_set_default_settings)"""
    return [(f"a{j}.info", a._obj) for j, a in enumerate(args)
            if type(a).__name__ == "CArgObject" and isinstance(a._obj, (capi.ScsInfo, capi.ScsSettings))]


def _current_test():
    t = os.environ["PYTEST_CURRENT_TEST"].rsplit(" ", 1)[0]
    path, name = t.split("::", 1)
    return os.path.splitext(os.path.basename(path))[0], name


class _Session:
    def __init__(self):
        self.record_dir = os.environ.get("SCS_RECORD_REFERENCE")
        self.stores = {}     # module -> {key: array}
        self.counts = {}     # (module, test) -> calls so far

    def store(self, module):
        if module not in self.stores:
            if self.record_dir:
                self.stores[module] = {}
            else:
                with np.load(os.path.join(GOLDEN_DIR, module + ".npz")) as z:
                    index = json.loads(z["index"].tobytes())
                    blobs = {"f8": z["f8"], "u1": z["u1"]}
                self.stores[module] = {k: blobs[dt][o:o + n].reshape(shape) for k, (dt, o, n, shape) in index.items()}
        return self.stores[module]

    def next_key(self):
        module, test = _current_test()
        i = self.counts.get((module, test), 0)
        self.counts[(module, test)] = i + 1
        return self.store(module), f"{test}|{i}|"

    def save(self):
        if not self.record_dir:
            return
        os.makedirs(self.record_dir, exist_ok=True)
        for module, st in self.stores.items():
            index, parts = {}, {"f8": [], "u1": []}
            used = {"f8": 0, "u1": 0}
            for k, v in st.items():
                if v.dtype.kind == "U":   # function tags
                    v = np.frombuffer(str(v).encode(), dtype=np.uint8)
                    k = k + "@s"
                dt = "u1" if v.dtype == np.uint8 else "f8"
                index[k] = (dt, used[dt], int(v.size), list(v.shape))
                parts[dt].append(v.astype(dt).ravel())
                used[dt] += v.size
            np.savez_compressed(os.path.join(self.record_dir, module + ".npz"),
                                index=np.frombuffer(json.dumps(index).encode(), dtype=np.uint8),
                                **{dt: np.concatenate(p) if p else np.zeros(0, dt) for dt, p in parts.items()})


SESSION = _Session()


class _Function:
    def __init__(self, build, name):
        object.__setattr__(self, "_build", build)
        object.__setattr__(self, "_name", name)

    def __setattr__(self, attr, value):  # restype / argtypes: only the real library needs them
        if self._build.lib is not None:
            setattr(getattr(self._build.lib, self._name), attr, value)

    def __call__(self, *args):
        store, key = SESSION.next_key()
        tag = f"{self._build.kind}:{self._name}"
        if self._build.lib is not None:
            before = {s: arr.copy() for s, arr in _slots(args)}
            ret = getattr(self._build.lib, self._name)(*args)
            store[key + "fn"] = np.array(tag)
            if isinstance(ret, (int, float)):   # handles are ints as well: addresses below 2^53
                store[key + ("ret_i" if isinstance(ret, int) else "ret")] = np.array(float(ret))
            for s, arr in _slots(args):
                if not np.array_equal(arr, before[s], equal_nan=True):
                    for suffix, v in _pack(arr, self._build.whole).items():
                        store[key + s + suffix] = v
            for s, info in _infos(args):
                store[key + s] = np.frombuffer(bytes(info), dtype=np.uint8).copy()
            return ret
        assert key + "fn@s" in store, f"no recorded reference call {key} (re-record tests/golden/reference/)"
        recorded = store[key + "fn@s"].tobytes().decode()
        assert recorded == tag, (key, recorded, tag)
        for s, arr in _slots(args):
            if key + s in store:
                _unpack(store, key + s, arr)
        for s, info in _infos(args):
            raw = store[key + s].tobytes()
            C.memmove(C.addressof(info), raw, len(raw))
        if key + "ret_i" in store:
            return int(store[key + "ret_i"].item())
        return store[key + "ret"].item() if key + "ret" in store else None


class Reference:
    """The reference build `kind` (see BUILDS): the real library while recording, its recorded answers otherwise.
    whole=True stores every array whole, for tests that use all entries of the reference's results."""

    def __init__(self, kind="ref", whole=False):
        self.kind = kind
        self.whole = whole
        self.lib = None
        if SESSION.record_dir:
            path = os.path.join(REF_DIR, BUILDS[kind])
            if not os.path.exists(path):
                raise RuntimeError(f"recording needs the reference build {path} (make -C oracle ref)")
            self.lib = capi.load_reference(path)

    def __getattr__(self, name):
        return _Function(self, name)

    def written_file(self, path):
        """a file the previous call wrote (log_csv_filename): recorded byte for byte, written back on replay"""
        store, key = SESSION.next_key()
        if self.lib is not None:
            with open(path, "rb") as f:
                store[key + "file"] = np.frombuffer(f.read(), dtype=np.uint8).copy()
        else:
            with open(path, "wb") as f:
                f.write(store[key + "file"].tobytes())
