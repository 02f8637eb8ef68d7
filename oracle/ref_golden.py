"""Recorded outputs of the reference's own CUDA kernels (oracle/ref_cuda.py) for the GPU parity tests.

The parity tests compare the product with the reference's kernels on seeded scenes.  The reference is not part of this
repository, so the tests do not run it: `RefDirectBA` here has the interface of `ref_cuda.RefDirectBA` and plays back what
the reference returned for the same calls, stored per test in tests/golden/ref/<module>/<test>.npz.

Every call is keyed by (instance of RefDirectBA within the test, call index, method), and a digest of its array and scalar
arguments is stored with it: playing a call back with other arguments than were recorded fails, so a test cannot pass
against reference values computed for different inputs.  Arrays of up to FULL_LIMIT elements are stored whole.  Of larger
ones a fixed part is kept -- images (more than 16 rows): a band of central rows of about BAND elements; arrays of a few
rows (surfel rows): SAMPLE seeded columns, all rows of each; vectors: the first and last HEAD_TAIL elements and SAMPLE
seeded ones in between -- and they play back as numpy masked arrays whose other elements are masked, so that maxima, means
and counts in the tests run over the stored elements.  Compare them with `equal()`, not `np.array_equal`, and crop images
to `kept_rows()` before neighbourhood operations.

    BADBA_RECORD_REF=1 python -m pytest tests -m gpu     # re-record: needs a GPU and oracle/_ref (oracle/build_ref.sh)

When recording, each call runs on the reference's kernels and the test sees the value as it will be played back.
"""
from __future__ import annotations

import atexit
import ctypes as C
import hashlib
import os
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN_DIR = os.path.join(ROOT, "tests", "golden", "ref")
RECORD = os.environ.get("BADBA_RECORD_REF") == "1"
FULL_LIMIT, HEAD_TAIL, SAMPLE, BAND = 16384, 512, 4096, 8192

_tapes: dict[str, dict] = {}      # module/test -> {key: array}
_instances: dict[str, int] = {}   # test id -> RefDirectBA instances created so far


def available() -> bool:
    """Playback needs no GPU; recording needs the reference's library."""
    if RECORD:
        from oracle import ref_cuda
        return ref_cuda.available()
    return True


def _current_test():
    """'<module>/<test name with parameters>' of the running pytest test."""
    node = os.environ["PYTEST_CURRENT_TEST"].rsplit(" ", 1)[0]
    path, name = node.split("::", 1)
    return os.path.splitext(os.path.basename(path))[0] + "/" + name


def _tape(test):
    if test not in _tapes:
        path = os.path.join(GOLDEN_DIR, test + ".npz")
        if RECORD:
            _tapes[test] = {}
            atexit.register(_save, test)
        else:
            if not os.path.exists(path):
                raise FileNotFoundError(f"{path}: no recorded reference outputs for this test (see oracle/ref_golden.py)")
            with np.load(path) as z:
                _tapes[test] = dict(z)
    return _tapes[test]


def _save(test):
    path = os.path.join(GOLDEN_DIR, test + ".npz")
    os.makedirs(os.path.dirname(path), exist_ok=True)
    np.savez_compressed(path, **_tapes[test])


def _digest(args, kwargs):
    """sha1 over the array and scalar arguments of a call (exact bits, dtype and shape of arrays)."""
    h = hashlib.sha1()
    for name, a in [(str(i), a) for i, a in enumerate(args)] + sorted(kwargs.items()):
        h.update(name.encode())
        if a is None or isinstance(a, (bool, int, float, str, np.generic, np.ndarray, list, tuple)):
            a = np.asarray(a) if a is not None else np.zeros(0)
            h.update(repr((a.dtype.str, a.shape)).encode())
            h.update(np.ascontiguousarray(a).tobytes())
        else:
            h.update(type(a).__name__.encode())
    return np.frombuffer(h.digest(), np.uint8)


def sample_index(size):
    """The flat indices kept of an array of `size` elements (deterministic in `size`)."""
    if size <= FULL_LIMIT:
        return np.arange(size)
    mid = np.random.default_rng(size).choice(np.arange(HEAD_TAIL, size - HEAD_TAIL), SAMPLE, replace=False)
    return np.unique(np.concatenate([np.arange(HEAD_TAIL), mid, np.arange(size - HEAD_TAIL, size)]))


def _columns(n):
    """The columns kept of an array of a few rows and `n` columns (deterministic in `n`)."""
    return np.sort(np.random.default_rng(n).choice(n, min(n, SAMPLE), replace=False))


def _band(shape):
    """The rows kept of an image of `shape`: about BAND elements around the middle row."""
    n = max(1, min(shape[0], BAND // int(np.prod(shape[1:]))))
    r0 = (shape[0] - n) // 2
    return slice(r0, r0 + n)


def kept_rows(a):
    """The rows of a played-back image that hold stored values (all rows of an array stored whole)."""
    if not np.ma.isMaskedArray(a):
        return slice(0, a.shape[0])
    rows = np.flatnonzero(~np.ma.getmaskarray(a).reshape(a.shape[0], -1).all(axis=1))
    return slice(int(rows[0]), int(rows[-1]) + 1)


def _encode(v, key, out):
    if v is None:
        out[key + ":none"] = np.zeros(0, np.int8)
    elif isinstance(v, tuple):
        out[key + ":tuple"] = np.array(len(v))
        for i, x in enumerate(v):
            _encode(x, f"{key}.{i}", out)
    elif isinstance(v, C.Structure):
        out[key + ":struct"] = np.array([f for f, _ in v._fields_])
        for f, _ in v._fields_:
            x = getattr(v, f)
            _encode(np.array(x[:]) if isinstance(x, C.Array) else x, f"{key}.{f}", out)
    elif isinstance(v, np.ndarray) and v.size > FULL_LIMIT and v.ndim >= 2 and v.shape[0] > 16:
        rows = _band(v.shape)
        out[key + ":band"] = np.ascontiguousarray(v[rows])
        out[key + ":shape"] = np.array(v.shape)
    elif isinstance(v, np.ndarray) and v.size > FULL_LIMIT and v.ndim == 2:
        out[key + ":columns"] = np.ascontiguousarray(v[:, _columns(v.shape[1])])
        out[key + ":shape"] = np.array(v.shape)
    elif isinstance(v, np.ndarray) and v.size > FULL_LIMIT:
        out[key + ":sampled"] = np.ascontiguousarray(v).reshape(-1)[sample_index(v.size)]
        out[key + ":shape"] = np.array(v.shape)
    elif isinstance(v, np.ndarray):
        out[key + ":array"] = v
    else:
        out[key + ":scalar"] = np.array(v)


def _decode(tape, key):
    if key + ":none" in tape:
        return None
    if key + ":tuple" in tape:
        return tuple(_decode(tape, f"{key}.{i}") for i in range(int(tape[key + ":tuple"])))
    if key + ":struct" in tape:
        return types.SimpleNamespace(**{str(f): _decode(tape, f"{key}.{f}") for f in tape[key + ":struct"]})
    if key + ":band" in tape:
        shape = tuple(int(s) for s in tape[key + ":shape"])
        data, mask = np.zeros(shape, tape[key + ":band"].dtype), np.ones(shape, bool)
        data[_band(shape)], mask[_band(shape)] = tape[key + ":band"], False
        return np.ma.MaskedArray(data, mask)
    if key + ":columns" in tape:
        shape = tuple(int(s) for s in tape[key + ":shape"])
        data, mask = np.zeros(shape, tape[key + ":columns"].dtype), np.ones(shape, bool)
        data[:, _columns(shape[1])], mask[:, _columns(shape[1])] = tape[key + ":columns"], False
        return np.ma.MaskedArray(data, mask)
    if key + ":sampled" in tape:
        shape = tuple(int(s) for s in tape[key + ":shape"])
        kept = tape[key + ":sampled"]
        data = np.zeros(int(np.prod(shape)), kept.dtype)
        mask = np.ones(data.size, bool)
        idx = sample_index(data.size)
        data[idx], mask[idx] = kept, False
        return np.ma.MaskedArray(data.reshape(shape), mask.reshape(shape))
    if key + ":array" in tape:
        return tape[key + ":array"].copy()
    if key + ":scalar" in tape:
        return tape[key + ":scalar"].item()
    raise KeyError(f"no recorded reference output {key!r}: re-record with BADBA_RECORD_REF=1 (see oracle/ref_golden.py)")


def equal(a, b):
    """np.array_equal over the elements a recorded (possibly sampled) reference array kept."""
    a, b = np.ma.asarray(a), np.ma.asarray(b)
    if a.shape != b.shape:
        return False
    mask = np.ma.getmaskarray(a) | np.ma.getmaskarray(b)
    return bool(np.array_equal(np.ma.getdata(a)[~mask], np.ma.getdata(b)[~mask]))


class RefDirectBA:
    """ref_cuda.RefDirectBA played back from (or, with BADBA_RECORD_REF=1, recorded into) tests/golden/ref.  The constructor's
    scene is not digested: the tests build it from a seeded configuration."""

    def __init__(self, scene, *args, **kwargs):
        test = _current_test()
        n = _instances.get(test, 0)
        _instances[test] = n + 1
        self._prefix = str(n)
        self._calls = 0
        self._tape = _tape(test)
        self._live = None
        if RECORD:
            from oracle import ref_cuda
            self._live = ref_cuda.RefDirectBA(scene, *args, **kwargs)

    def __getattr__(self, name):
        if name.startswith("_"):
            raise AttributeError(name)

        def call(*args, **kwargs):
            key = f"{self._prefix}|{self._calls}|{name}"
            self._calls += 1
            digest = _digest(args, kwargs)
            if RECORD:
                _encode(getattr(self._live, name)(*args, **kwargs), key, self._tape)
                self._tape[key + ":args"] = digest
            if key + ":args" not in self._tape:
                raise KeyError(f"no recorded reference output {key!r}: re-record with BADBA_RECORD_REF=1 (see oracle/ref_golden.py)")
            if not np.array_equal(self._tape[key + ":args"], digest):
                raise AssertionError(f"reference call {key!r} played back with other arguments than were recorded")
            return _decode(self._tape, key)
        return call

    def close(self):
        if self._live is not None:
            self._live.close()
