"""Recorded answers of the executed reference (oracle/_ref) for the tests that compare against it.

The reference binaries are built from the reference tree's sources, which a checkout of this repository does not carry.
tests/golden/make_live_ref_vectors.py runs those tests once against the live binaries with a `Recorder` around them and
stores every answer in tests/golden/live_ref_vectors.npz; everywhere else a `Replay` gives the same answers to the same
calls, in the same order, and checks that each call is the recorded one (method name and a digest of the arguments).

What is kept of an answer: integer arrays, and complex arrays of at most WHOLE elements, whole.  A larger complex array
is cut into STRATA equal strata and one element at a fixed, seeded position in each stratum is kept, together with the
last element (the tail of an uneven split) and the element of largest magnitude; the replay returns a masked array in
which only those elements are present, and numpy's masked reductions then compare the product or the oracle there.  So
every buffer of every device is compared in each 1/STRATA-th of its length, and any difference that covers a stratum of a
buffer is seen."""
import hashlib
import json
import os

import numpy as np

PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "live_ref_vectors.npz")
WHOLE = 64
STRATA = 32


def _test_id():
    return os.environ.get("PYTEST_CURRENT_TEST", "").split(" ")[0]


def _positions(n, peak):
    """kept elements of an n-element array whose largest-magnitude element is at `peak`"""
    edges = np.linspace(0, n, STRATA + 1).astype(np.int64)
    rng = np.random.default_rng(n)
    picks = [int(rng.integers(a, b)) for a, b in zip(edges[:-1], edges[1:])]
    return np.unique(picks + [n - 1, peak])


def _digest(args, answers):
    """method arguments as text: arrays by content, except answers of the reference (in a replay: the arrays standing for
    them), whose stored form is not their content"""
    def desc(x):
        if isinstance(x, np.ndarray):
            if id(x) in answers:
                return "answer"
            return "%s%s:%s" % (x.dtype.str, x.shape, hashlib.sha1(np.ascontiguousarray(x).tobytes()).hexdigest()[:16])
        if isinstance(x, (list, tuple)):
            return "[" + ",".join(desc(v) for v in x) + "]"
        if isinstance(x, (bool, int, float, str, type(None), np.integer, np.floating)):
            return repr(x.item() if isinstance(x, (np.integer, np.floating)) else x)
        return type(x).__name__ + desc([v for v in vars(x).values() if isinstance(v, (int, np.integer))])
    return hashlib.sha1(desc(list(args)).encode()).hexdigest()[:16]


def _put(pools, v):
    """append v to the pool of its dtype; returns its offset there"""
    pool = pools.setdefault(v.dtype.str, [])
    off = sum(x.size for x in pool)
    pool.append(v.reshape(-1))
    return off


def _pack(v, pools, answers):
    if isinstance(v, np.ndarray):
        answers[id(v)] = v
        if v.dtype.kind == "i" and np.abs(v).max(initial=0) < 2 ** 31:
            v = v.astype(np.int32)
        if v.dtype.kind != "c" or v.size <= WHOLE:
            return {"a": _put(pools, v), "t": v.dtype.str, "z": list(v.shape)}
        flat = v.reshape(-1)
        peak = int(np.argmax(np.abs(flat)))
        return {"s": _put(pools, flat[_positions(flat.size, peak)]), "p": peak, "t": v.dtype.str, "z": list(v.shape)}
    if isinstance(v, (list, tuple)):
        return {"l": [_pack(x, pools, answers) for x in v]}
    if isinstance(v, (np.integer, np.floating)):
        return v.item()
    return v


def _unpack(d, z):
    if isinstance(d, dict):
        n = int(np.prod(d["z"])) if "z" in d else 0
        if "a" in d:
            return z[d["t"]][d["a"]: d["a"] + n].reshape(d["z"])
        if "s" in d:
            pos = _positions(n, d["p"])
            data = np.zeros(n, dtype=np.dtype(d["t"]))
            mask = np.ones(n, dtype=bool)
            data[pos] = z[d["t"]][d["s"]: d["s"] + pos.size]
            mask[pos] = False
            return np.ma.masked_array(data, mask).reshape(d["z"])
        return [_unpack(x, z) for x in d["l"]]
    return d


class Recorder:
    """Wraps a live reference binding; every method call's answer is kept under (test id, call number)."""

    def __init__(self, live, store):
        self._live, self._store = live, store

    def __getattr__(self, name):
        fn = getattr(self._live, name)

        def call(*args, **kwargs):
            answers = self._store.setdefault("answers", {})    # also keeps the answers alive, so that their ids stay unique
            h = _digest(list(args) + sorted(kwargs.items()), answers)
            out = fn(*args, **kwargs)
            calls = self._store.setdefault("calls", {}).setdefault(_test_id(), [])
            calls.append({"m": name, "h": h, "r": _pack(out, self._store.setdefault("pools", {}), answers)})
            return out
        return call


def save(store, path=PATH):
    calls = np.frombuffer(json.dumps(store.get("calls", {}), separators=(",", ":")).encode(), dtype=np.uint8)
    np.savez_compressed(path, _calls=calls, **{dt: np.concatenate(pool) for dt, pool in store.get("pools", {}).items()})


class Replay:
    """Gives the recorded answers back in call order, after checking that each call is the one that was recorded."""

    def __init__(self, path=PATH):
        with np.load(path) as z:
            self._z = {k: z[k] for k in z.files}
        self._calls = json.loads(self._z["_calls"].tobytes().decode())
        self._next = {}
        self._answers = {}          # the arrays handed out, kept alive so that their ids stay unique

    def _keep(self, v):
        if isinstance(v, np.ndarray):
            self._answers[id(v)] = v
        elif isinstance(v, list):
            for x in v:
                self._keep(x)
        return v

    def __getattr__(self, name):
        def call(*args, **kwargs):
            tid = _test_id()
            k = self._next.get(tid, 0)
            self._next[tid] = k + 1
            rec = self._calls.get(tid, [])
            assert k < len(rec), f"{tid}: no recorded answer for call {k} ({name}); rerun tests/golden/make_live_ref_vectors.py"
            h = _digest(list(args) + sorted(kwargs.items()), self._answers)
            assert (rec[k]["m"], rec[k]["h"]) == (name, h), \
                f"{tid}: call {k} is {name} with other arguments than the recorded {rec[k]['m']}; rerun tests/golden/make_live_ref_vectors.py"
            return self._keep(_unpack(rec[k]["r"], self._z))
        return call


def reference(live_factory, build):
    """The live binding when the reference binaries are present (wrapped in a Recorder while
    tests/golden/make_live_ref_vectors.py records), else the replay of the recorded answers."""
    if build() is not None:
        live = live_factory()
        store = RECORDING.get("store")
        return Recorder(live, store) if store is not None else live
    return Replay()


RECORDING = {}
