"""The reference's own templates (oracle/_ref/libnvbio_ref.so) where they are built, their stored answers everywhere else.

`reference()` returns the live library when it exists, else a replayer of tests/golden/ref_calls.pkl.gz: every call made by the
CPU tests against the reference was recorded there with its result, keyed by a digest of the method name and all its arguments
(plus the new contents of any dict argument the call updates in place, such as a windowed DP's state), so a test keeps
comparing against the reference's own outputs on machines without an nvbio tree.  A call whose inputs were never recorded
fails the test (the inputs changed: record again).  To record, build oracle/_ref and run the CPU tests with
NVB_RECORD_REF=1; the calls are merged into the stored file."""
import gzip
import hashlib
import os
import pickle

import numpy as np

from oracle import orc

PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "ref_calls.pkl.gz")


def _digest(name, args, kwargs):
    h = hashlib.sha256(name.encode())

    def feed(v):
        if isinstance(v, np.ndarray):
            h.update(("nd%s%s" % (v.dtype.str, v.shape)).encode())
            h.update(np.ascontiguousarray(v).tobytes())
        elif isinstance(v, dict):
            h.update(b"{")
            for k in sorted(v):
                h.update(repr(k).encode()); feed(v[k])
            h.update(b"}")
        elif isinstance(v, (list, tuple)):
            h.update(b"(")
            for x in v:
                feed(x)
            h.update(b")")
        elif isinstance(v, (np.integer, np.floating)):
            h.update(repr(v.item()).encode())
        else:
            h.update(repr(v).encode())
    feed(list(args)); feed(dict(kwargs))
    return h.hexdigest()


def _load():
    if not os.path.exists(PATH):
        return {}
    with gzip.open(PATH, "rb") as f:
        return pickle.load(f)


class _Recorder:
    def __init__(self, ref):
        self.ref, self.calls = ref, {}

    def __getattr__(self, name):
        fn = getattr(self.ref, name)
        if name in ("set_num_threads", "num_threads"):
            return fn

        def call(*args, **kwargs):
            key = _digest(name, args, kwargs)
            dicts = {i: a for i, a in enumerate(list(args) + list(kwargs.values())) if isinstance(a, dict)}
            before = {i: _digest("", (a,), {}) for i, a in dicts.items()}
            r = fn(*args, **kwargs)
            updated = {i: {k: np.copy(v) for k, v in a.items()} for i, a in dicts.items() if _digest("", (a,), {}) != before[i]}
            self.calls[key] = (r, updated)
            return r
        return call

    def save(self):
        calls = _load()
        calls.update(self.calls)
        with gzip.open(PATH, "wb", compresslevel=9) as f:
            pickle.dump(calls, f, protocol=4)


class _Replay:
    kind = "reference"

    def __init__(self, calls):
        self.calls = calls

    def set_num_threads(self, t):
        pass

    def __getattr__(self, name):
        def call(*args, **kwargs):
            key = _digest(name, args, kwargs)
            assert key in self.calls, "no stored reference answer for this %s call (inputs changed? record again)" % name
            r, updated = self.calls[key]
            allargs = list(args) + list(kwargs.values())
            for i, state in updated.items():
                for k, v in state.items():
                    allargs[i][k][...] = v
            return r
        return call


_recorders = []


def live_exports(symbols):
    """whether oracle/_ref/libnvbio_ref.so is built and exports every one of `symbols` (an _ref/ built from an older oracle/ref_shim.cpp,
    used as is where no nvbio tree is at hand to rebuild it, lacks the newer entry points)"""
    if not orc.Ref.available():
        return False
    lib = orc.Ref().lib
    return all(hasattr(lib, s) for s in symbols)


def reference(symbols=()):
    """the live reference library (recording when NVB_RECORD_REF is set) where it is built and exports `symbols`, else the stored
    answers"""
    if live_exports(symbols):
        if os.environ.get("NVB_RECORD_REF"):
            _recorders.append(_Recorder(orc.Ref()))
            return _recorders[-1]
        return orc.Ref()
    calls = _load()
    assert calls, "neither oracle/_ref/libnvbio_ref.so nor %s is present" % PATH
    return _Replay(calls)


def save_recordings():
    for r in _recorders:
        r.save()
    _recorders.clear()
