"""oracle -- the CPU checker for the GPU Aho-Corasick search path.

TEST INFRASTRUCTURE ONLY.  Importable from ``tests/``, ``__graft_entry__.smoke()``
and ``bench.py``'s ``cpu_baseline`` / ``--impl reference`` legs; nothing under
``pyahocorasick_b200/`` imports this package (tests/test_no_oracle_in_product.py
enforces it).

Two checkers live here:

* ``OracleAutomaton`` -- ctypes wrapper around ``liboracle_ac.so``, the plain-C
  restatement in ``oracle/ac_oracle.c`` (cites the reference file:line it follows).
* ``ref_module(flavour)`` -- the UNMODIFIED reference extension compiled from
  ``/root/reference/src/pyahocorasick.c`` into ``oracle/_ref/<flavour>/`` by
  ``oracle/Makefile`` (``make ref``).  It travels to the GPU box as a prebuilt file.

Parity status: pinned (see tests/test_oracle.py and tests/golden/).
"""
from __future__ import annotations

import ctypes
import importlib.machinery
import importlib.util
import os
import subprocess
import sysconfig

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "liboracle_ac.so")
_REF_DIR = os.path.join(_HERE, "_ref")

EMPTY, TRIE, AHOCORASICK = 0, 1, 2


def build(ref: bool = True) -> None:
    """Compile the C restatement and, when /root/reference is present, the reference."""
    subprocess.check_call(["make", "-s", "-C", _HERE, "liboracle_ac.so"])
    if ref and os.path.exists("/root/reference/src/pyahocorasick.c"):
        subprocess.check_call(["make", "-s", "-C", _HERE, "ref"])


_lib = None


def lib() -> ctypes.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(_LIB_PATH):
        build(ref=False)
    L = ctypes.CDLL(_LIB_PATH)
    vp, i64, i32p, i64p = ctypes.c_void_p, ctypes.c_int64, ctypes.POINTER(ctypes.c_int32), ctypes.POINTER(ctypes.c_int64)
    u32p, u8p = ctypes.POINTER(ctypes.c_uint32), ctypes.POINTER(ctypes.c_uint8)
    L.orc_new.restype = vp
    L.orc_free.argtypes = [vp]
    for name in ("orc_kind", "orc_count", "orc_longest", "orc_version"):
        getattr(L, name).argtypes = [vp]
        getattr(L, name).restype = ctypes.c_int
    L.orc_nodes.argtypes = [vp]
    L.orc_nodes.restype = i64
    L.orc_add_word.argtypes = [vp, u32p, i64, i64]
    L.orc_add_word.restype = ctypes.c_int
    L.orc_make_automaton.argtypes = [vp]
    L.orc_make_automaton.restype = ctypes.c_int
    L.orc_find_all.argtypes = [vp, u32p, i64, i64, i64p, i64p, i64]
    L.orc_find_all.restype = i64
    L.orc_iter_long.argtypes = [vp, u32p, i64, i64, i64p, i64p, i64]
    L.orc_iter_long.restype = i64
    L.orc_iter_new.argtypes = [vp, u32p, i64, i64, ctypes.c_int]
    L.orc_iter_new.restype = vp
    L.orc_iter_free.argtypes = [vp]
    L.orc_iter_next.argtypes = [vp, i64p, i64p]
    L.orc_iter_next.restype = ctypes.c_int
    L.orc_iter_set.argtypes = [vp, u32p, i64, ctypes.c_int]
    L.orc_scan_batch_bytes.argtypes = [vp, u8p, i64p, i64, i32p, i64]
    L.orc_scan_batch_bytes.restype = i64
    L.orc_widen_bytes.argtypes = [u8p, i64, u32p]
    _lib = L
    return L


def _letters(obj) -> np.ndarray:
    """Turn a key / haystack into the reference's letter array.

    bytes  -> sign-extended 16-bit letters (bytes flavour, src/utils.c:199-202)
    str    -> UCS-4 code points            (unicode flavour, src/utils.c:154-169)
    tuple  -> integers as given            (KEY_SEQUENCE, src/utils.c:239-278)
    """
    if isinstance(obj, (bytes, bytearray, memoryview)):
        a = np.frombuffer(bytes(obj), dtype=np.int8).astype(np.int16).astype(np.uint16).astype(np.uint32)
    elif isinstance(obj, str):
        a = np.frombuffer(obj.encode("utf-32-le", "surrogatepass"), dtype=np.uint32).copy()
    else:
        a = np.asarray(list(obj), dtype=np.uint32)
    return np.ascontiguousarray(a)


def _p(a: np.ndarray, ct):
    return a.ctypes.data_as(ctypes.POINTER(ct))


class OracleAutomaton:
    """Integer-valued automaton (value = whatever int the caller passes, e.g. a key id)."""

    def __init__(self):
        self._L = lib()
        self._h = self._L.orc_new()
        self._keep = []

    def __del__(self):
        try:
            self._L.orc_free(self._h)
        except Exception:
            pass

    @property
    def kind(self):
        return self._L.orc_kind(self._h)

    def __len__(self):
        return self._L.orc_count(self._h)

    @property
    def longest_word(self):
        return self._L.orc_longest(self._h)

    @property
    def nodes_count(self):
        return self._L.orc_nodes(self._h)

    def add_word(self, key, value: int) -> bool:
        w = _letters(key)
        r = self._L.orc_add_word(self._h, _p(w, ctypes.c_uint32), len(w), int(value))
        if r < 0:
            raise MemoryError
        return bool(r)

    def make_automaton(self):
        r = self._L.orc_make_automaton(self._h)
        if r < 0:
            raise MemoryError
        return None if r == 1 else False

    def find_all(self, text, start=0, end=None):
        """[(end_index, value)] in the reference's order, or None if not built."""
        w = _letters(text)
        if end is None:
            end = len(w)
        cap = 1024
        while True:
            idx = np.empty(cap, dtype=np.int64)
            val = np.empty(cap, dtype=np.int64)
            n = self._L.orc_find_all(self._h, _p(w, ctypes.c_uint32), start, end,
                                     _p(idx, ctypes.c_int64), _p(val, ctypes.c_int64), cap)
            if n < 0:
                return None
            if n <= cap:
                return list(zip(idx[:n].tolist(), val[:n].tolist()))
            cap = int(n)

    def iter(self, text, start=0, end=None, ignore_white_space=False):
        return OracleIter(self, text, start, end, ignore_white_space)

    def iter_long(self, text, start=0, end=None):
        """[(end_index, value)] of the longest-match variant (src/AutomatonSearchIterLong.c)."""
        w = _letters(text)
        if end is None:
            end = len(w)
        cap = 1024
        while True:
            idx = np.empty(cap, dtype=np.int64)
            val = np.empty(cap, dtype=np.int64)
            n = self._L.orc_iter_long(self._h, _p(w, ctypes.c_uint32), start, end,
                                      _p(idx, ctypes.c_int64), _p(val, ctypes.c_int64), cap)
            if n < 0:
                raise AttributeError("not an automaton yet")
            if n <= cap:
                return list(zip(idx[:n].tolist(), val[:n].tolist()))
            cap = int(n)

    def scan_batch_bytes(self, flat: np.ndarray, offsets: np.ndarray) -> np.ndarray:
        """(n,3) int32 records (hay_id, end_index, value) in scan order."""
        flat = np.ascontiguousarray(flat, dtype=np.uint8)
        offsets = np.ascontiguousarray(offsets, dtype=np.int64)
        n = len(offsets) - 1
        cap = max(1024, n)
        while True:
            out = np.empty((cap, 3), dtype=np.int32)
            tot = self._L.orc_scan_batch_bytes(self._h, _p(flat, ctypes.c_uint8), _p(offsets, ctypes.c_int64),
                                               n, _p(out, ctypes.c_int32), cap)
            if tot < 0:
                raise AttributeError("not an automaton")
            if tot <= cap:
                return out[:tot]
            cap = int(tot)


class OracleIter:
    def __init__(self, A: OracleAutomaton, text, start, end, ignore_ws):
        self._A = A
        self._L = A._L
        self._w = _letters(text)
        if end is None:
            end = len(self._w)
        self._it = self._L.orc_iter_new(A._h, _p(self._w, ctypes.c_uint32), start, end, int(bool(ignore_ws)))
        if not self._it:
            raise AttributeError("Not an Aho-Corasick automaton yet")

    def __del__(self):
        try:
            self._L.orc_iter_free(self._it)
        except Exception:
            pass

    def __iter__(self):
        return self

    def __next__(self):
        i = ctypes.c_int64()
        v = ctypes.c_int64()
        r = self._L.orc_iter_next(self._it, ctypes.byref(i), ctypes.byref(v))
        if r == 1:
            return (i.value, v.value)
        if r == -2:
            raise ValueError("underlaying automaton has changed, iterator is not valid anymore")
        raise StopIteration

    def set(self, text, reset=False):
        self._w = _letters(text)
        self._L.orc_iter_set(self._it, _p(self._w, ctypes.c_uint32), len(self._w), int(bool(reset)))


# ---------------------------------------------------------------------------
# the compiled reference
# ---------------------------------------------------------------------------
_ref_cache = {}


def ref_available(flavour: str = "bytes") -> bool:
    return os.path.exists(_ref_path(flavour))


def _ref_path(flavour: str) -> str:
    return os.path.join(_REF_DIR, flavour, "ahocorasick" + sysconfig.get_config_var("EXT_SUFFIX"))


def ref_module(flavour: str = "bytes"):
    """Import the unmodified reference extension (flavour 'bytes' or 'unicode')."""
    if flavour in _ref_cache:
        return _ref_cache[flavour]
    path = _ref_path(flavour)
    if not os.path.exists(path):
        raise ImportError(f"reference extension not built: {path} (run `make -C oracle ref` where /root/reference exists)")
    loader = importlib.machinery.ExtensionFileLoader("ahocorasick", path)
    spec = importlib.util.spec_from_file_location("ahocorasick", path, loader=loader)
    mod = importlib.util.module_from_spec(spec)
    loader.exec_module(mod)
    _ref_cache[flavour] = mod
    return mod


def ref_scan_batch(A, haystacks) -> list:
    """[(hay_id, end_index, value)] by looping the reference's iter() -- the differential oracle."""
    out = []
    for h, hay in enumerate(haystacks):
        for e, v in A.iter(hay):
            out.append((h, e, v))
    return out
