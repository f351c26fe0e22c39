"""The reference extension's recorded answers, so that the differential tests compare with the reference wherever they run.

The differential tests are seeded: they ask the reference (WojciechMula/pyahocorasick, compiled into oracle/_ref/) the
same questions in the same order on every run.  `reference(flavour)` returns a stand-in for the reference module that
answers every interaction a test has with it -- attribute reads, calls, iteration, len(), `in` -- from
tests/golden/reference_calls.json.xz, where the test's id keys the answers the real extension gave, in order.  The
questions (what was asked and with which arguments; for a path argument the file's name and contents) are chained into
one digest, stored with every 32nd answer and with every answer to a question with long byte strings or files -- the
arguments that come from the drop-in's own output, its pickles and save files; all others come from the tests' seeds.
A replay that asks something other than what was recorded fails (a test edited without re-recording).  Files the
reference wrote (save()) are recorded and written again; callbacks it called (find_all(), save() / load()
serialisers) are called again with the recorded arguments.

Tests that compare whole batches keep a digest of the reference's records instead (`records_digest`,
tests/golden/reference_digests.json).

ACB_RECORD_REFERENCE=1, where oracle/_ref is built, runs the real extension and rewrites the entries of the tests
that ran (tests/golden/record_reference.py for the ones that need a GPU to run).
"""
import atexit
import base64
import builtins
import hashlib
import json
import lzma
import os

import numpy as np

_GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CALLS = os.path.join(_GOLDEN, "reference_calls.json.xz")
DIGESTS = os.path.join(_GOLDEN, "reference_digests.json")
RECORD = os.environ.get("ACB_RECORD_REFERENCE") == "1"

_calls = None          # test id -> recorded steps
_digests = None        # name -> {"records": n, "sha256": hex}
_sessions = {}
_recorded_calls = {}
_recorded_digests = {}


def test_id() -> str:
    """`test_module.py::test_name[params]` of the running test (pytest sets PYTEST_CURRENT_TEST)"""
    cur = os.environ.get("PYTEST_CURRENT_TEST", "")
    return os.path.basename(cur.rsplit(" (", 1)[0])


def _load_calls():
    global _calls
    if _calls is None:
        with lzma.open(CALLS, "rt", encoding="utf-8") as f:
            _calls = json.load(f)
    return _calls


def _load_digests():
    global _digests
    if _digests is None:
        with open(DIGESTS) as f:
            _digests = json.load(f)
    return _digests


def _sha(b: bytes) -> str:
    return hashlib.sha256(b).hexdigest()


def _canon(x):
    """what identifies an argument: values as they are, large byte strings by their hash, paths by name and contents"""
    if isinstance(x, _Proxy):
        return {"h": object.__getattribute__(x, "_h")}
    if isinstance(x, np.generic):
        x = x.item()
    if x is None or isinstance(x, (bool, int, float)):
        return x
    if isinstance(x, str):
        if x.startswith(os.sep):
            return {"path": os.path.basename(x), "sha256": _sha(open(x, "rb").read()) if os.path.isfile(x) else None}
        return x
    if isinstance(x, (bytes, bytearray)):
        return {"b": base64.b64encode(x).decode()} if len(x) <= 256 else {"bsha": _sha(bytes(x))}
    if isinstance(x, (tuple, list)):
        return {"t" if isinstance(x, tuple) else "l": [_canon(v) for v in x]}
    if isinstance(x, dict):
        return {"d": [[_canon(k), _canon(v)] for k, v in x.items()]}
    if callable(x):
        return {"fn": getattr(x, "__qualname__", type(x).__name__)}
    return {"repr": repr(x)}


def _question(h, kind, name, args, kw):
    """(canonical question, whether it carries data from outside the test's seed: long byte strings, files)"""
    q = json.dumps([h, kind, name, _canon(tuple(args)), _canon(dict(kw))], sort_keys=True)
    return q, '"bsha"' in q or '"path"' in q


CHECK_EVERY = 32


class _Session:
    """the answers of one test, in the order it asks for them"""

    def __init__(self, tid):
        self.tid = tid
        self.objs = {}                      # handle -> the extension's object (recording)
        self.n_handles = 0
        self.pos = 0
        self.chain = hashlib.sha256()
        if RECORD:
            self.rec = _recorded_calls[tid] = {"data": [], "steps": []}
        else:
            rec = _load_calls().get(tid)
            if rec is None:
                raise LookupError(f"{tid}: no recorded answers of the reference in {CALLS} "
                                  "(record them with ACB_RECORD_REFERENCE=1 where oracle/_ref is built)")
            self.rec = rec
        self.steps = self.rec["steps"]
        self.data_attrs = set(self.rec["data"])     # attributes that are values; any other attribute is a method

    # values cross as JSON: a value of the extension that is not plain data becomes a handle (a stand-in)
    def enc(self, x):
        if x is None or isinstance(x, (bool, int, float, str)):
            return x
        if isinstance(x, (bytes, bytearray)):
            return {"b": base64.b64encode(x).decode()}
        if isinstance(x, tuple):
            return {"t": [self.enc(v) for v in x]}
        if isinstance(x, list):
            return [self.enc(v) for v in x]
        if isinstance(x, dict):
            return {"d": [[self.enc(k), self.enc(v)] for k, v in x.items()]}
        h = self.n_handles
        self.n_handles += 1
        self.objs[h] = x
        return {"h": h}

    def dec(self, d):
        if isinstance(d, list):
            return [self.dec(v) for v in d]
        if not isinstance(d, dict):
            return d
        if "b" in d:
            return base64.b64decode(d["b"])
        if "t" in d:
            return tuple(self.dec(v) for v in d["t"])
        if "d" in d:
            return {self.dec(k): self.dec(v) for k, v in d["d"]}
        if not RECORD:
            self.n_handles = max(self.n_handles, d["h"] + 1)
        return _Proxy(self, d["h"])

    def attr(self, h, name):
        if RECORD and name not in self.data_attrs:
            if callable(getattr(self.objs[h], name)):
                return _Method(self, h, name)
            self.data_attrs.add(name)
            self.rec["data"].append(name)
        if name in self.data_attrs:
            return self.step(h, "getattr", name, (), {})
        return _Method(self, h, name)

    def step(self, h, kind, name, args, kw):
        q, external = _question(h, kind, name, args, kw)
        self.chain.update(q.encode())
        check = self.chain.hexdigest()[:16] if external or self.pos % CHECK_EVERY == 0 else None
        self.pos += 1
        if RECORD:
            return self._record(check, h, kind, name, args, kw)
        if self.pos > len(self.steps):
            raise AssertionError(f"{self.tid}: asks the reference more than was recorded (step {self.pos - 1})")
        st = self.steps[self.pos - 1]
        if check is not None and st.get("q") != check:
            raise AssertionError(f"{self.tid}: by step {self.pos - 1} the test has asked the reference something other than "
                                 f"what was recorded ({kind} {name or ''})")
        for i, b64 in st.get("files", []):
            with open(args[i], "wb") as f:
                f.write(base64.b64decode(b64))
        fn = next((a for a in args if callable(a) and not isinstance(a, _Proxy)), None)
        for cb in st.get("cb", []):
            fn(*self.dec(cb))
        if "exc" in st:
            tname, msg = st["exc"]
            exc_type = getattr(builtins, tname, None) or type(tname, (Exception,), {})
            raise exc_type(msg)
        return self.dec(st["r"])

    def _record(self, check, h, kind, name, args, kw):
        paths = [(i, a, open(a, "rb").read() if os.path.isfile(a) else None) for i, a in enumerate(args)
                 if isinstance(a, str) and a.startswith(os.sep)]
        cbs = []

        def wrap(a):
            if callable(a) and not isinstance(a, _Proxy):
                def cb(*cargs):
                    cbs.append(self.enc(cargs))
                    return a(*cargs)
                return cb
            return self.objs[object.__getattribute__(a, "_h")] if isinstance(a, _Proxy) else a
        target = self.objs[h]
        rargs = [wrap(a) for a in args]
        st = {} if check is None else {"q": check}
        self.steps.append(st)
        try:
            if kind == "getattr":
                r = getattr(target, name)
            elif kind == "method":
                r = getattr(target, name)(*rargs, **kw)
            elif kind == "call":
                r = target(*rargs, **kw)
            elif kind == "len":
                r = len(target)
            elif kind == "contains":
                r = rargs[0] in target
            elif kind == "iter":
                r = iter(target)
            elif kind == "next":
                r = next(target)
            else:
                r = target.__reduce__()
        except BaseException as e:
            st["exc"] = [type(e).__name__, str(e)]
            raise
        finally:
            if cbs:
                st["cb"] = cbs
            files = [[i, base64.b64encode(open(a, "rb").read()).decode()] for i, a, before in paths
                     if os.path.isfile(a) and open(a, "rb").read() != before]
            if files:
                st["files"] = files
        st["r"] = self.enc(r)
        return self.dec(st["r"])


class _Proxy:
    """stands in for the reference module or one of its objects (an Automaton, an iterator, a bound method)"""
    __slots__ = ("_s", "_h")

    def __init__(self, s, h):
        object.__setattr__(self, "_s", s)
        object.__setattr__(self, "_h", h)

    def _step(self, kind, name=None, args=(), kw=None):
        return object.__getattribute__(self, "_s").step(object.__getattribute__(self, "_h"), kind, name, args, kw or {})

    def __getattr__(self, name):
        return object.__getattribute__(self, "_s").attr(object.__getattribute__(self, "_h"), name)

    def __call__(self, *args, **kw):
        return self._step("call", None, args, kw)

    def __len__(self):
        return self._step("len")

    def __contains__(self, x):
        return self._step("contains", None, (x,))

    def __iter__(self):
        return self._step("iter")

    def __next__(self):
        return self._step("next")

    def __reduce__(self):
        return self._step("reduce")


class _Method:
    """a method of a stand-in: calling it is one question"""
    __slots__ = ("_s", "_h", "_name")

    def __init__(self, s, h, name):
        self._s, self._h, self._name = s, h, name

    def __call__(self, *args, **kw):
        return self._s.step(self._h, "method", self._name, args, kw)


def reference(flavour: str = "bytes"):
    """the reference module of `flavour` ('bytes' or 'unicode') for the running test"""
    tid = test_id()
    s = _sessions.get(tid)
    if s is None:
        s = _sessions[tid] = _Session(tid)
    h = "module:" + flavour
    if RECORD and h not in s.objs:
        import oracle
        s.objs[h] = oracle.ref_module(flavour)
    return _Proxy(s, h)


def records_digest(name: str, compute_reference_records) -> dict:
    """{"records": n, "sha256": ...} of the reference's (haystack, end_index, value) records for `name`;
    `compute_reference_records()` produces them (recording only)"""
    if RECORD:
        d = digest(compute_reference_records())
        _recorded_digests[name] = d
        return d
    return _load_digests()[name]


def reference_records(keys, haystacks) -> list:
    """[(haystack, end_index, key id)] by looping the real reference's iter() over byte haystacks (recording only)"""
    import oracle
    ref = oracle.ref_module("bytes")
    R = ref.Automaton(ref.STORE_INTS)
    for i, k in enumerate(keys):
        R.add_word(k, i)
    R.make_automaton()
    return oracle.ref_scan_batch(R, haystacks)


def digest(records) -> dict:
    a = np.ascontiguousarray(np.asarray(records, dtype=np.int64).reshape(-1, 3))
    return {"records": int(a.shape[0]), "sha256": _sha(a.tobytes())}


@atexit.register
def _save():
    if _recorded_calls:
        old = {}
        if os.path.exists(CALLS):
            with lzma.open(CALLS, "rt", encoding="utf-8") as f:
                old = json.load(f)
        old.update(_recorded_calls)
        with lzma.open(CALLS, "wt", encoding="utf-8", preset=9 | lzma.PRESET_EXTREME) as f:
            json.dump(old, f, sort_keys=True, separators=(",", ":"))
    if _recorded_digests:
        old = json.load(open(DIGESTS)) if os.path.exists(DIGESTS) else {}
        old.update(_recorded_digests)
        with open(DIGESTS, "w") as f:
            json.dump(old, f, indent=1, sort_keys=True)
            f.write("\n")
