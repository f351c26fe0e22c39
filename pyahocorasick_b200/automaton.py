"""`Automaton` -- the reference's Python surface (src/Automaton.c:1204-1256) on top of the
H100 C ABI (include/acb200.h).

Host side (this file + csrc/acb_host.cpp): keys, values, state machine EMPTY -> TRIE ->
AHOCORASICK, argument parsing and error behaviour of the reference.
Device side (csrc/acb_device.cu): every search -- `iter`, `find_all`, and the batch entry
`find_all_batch` -- runs on the GPU; there is no CPU search path in this package.

Reference semantics are cited as file:line relative to /root/reference.
"""
from __future__ import annotations

import codecs
import contextlib
import ctypes
import functools
import locale
import os
import operator
import pickle
import threading
import warnings
from typing import Any, Iterable, List, NamedTuple, Optional, Sequence, Tuple

import numpy as np

from . import _native as N


def _locked(method):
    """Run a method under the Automaton's GPU lock.  The native calls release the GIL (ctypes.CDLL) and a scan works
    in per-table scratch buffers, so two threads searching, or one searching while another changes the key set (which
    frees the device table), must not interleave; the reference gets the same guarantee from holding the GIL for the
    whole search (src/Automaton.c has no Py_BEGIN_ALLOW_THREADS)."""
    @functools.wraps(method)
    def wrapper(self, *args, **kwargs):
        with self._gpu_lock:
            return method(self, *args, **kwargs)
    return wrapper

# constants: src/Automaton.h:16-41, src/AutomatonItemsIter.h
EMPTY, TRIE, AHOCORASICK = 0, 1, 2
STORE_INTS, STORE_LENGTH, STORE_ANY = 10, 20, 30
KEY_STRING, KEY_SEQUENCE = 100, 200
MATCH_EXACT_LENGTH, MATCH_AT_MOST_PREFIX, MATCH_AT_LEAST_PREFIX = 0, 1, 2

_INT_MIN, _INT_MAX = -(2 ** 31), 2 ** 31 - 1
_LETTER_DTYPE = {1: np.uint8, 2: np.dtype("<u2"), 4: np.dtype("<u4")}


def _to_c_int(v: int) -> int:
    """Py_BuildValue("i", x) truncation of a Py_ssize_t (SURVEY A7)."""
    return ((int(v) + 2 ** 31) % 2 ** 32) - 2 ** 31


def _parse_c_int(x, name="an integer"):
    """PyArg 'i' format: int-like, must fit a C int."""
    if isinstance(x, float):
        raise TypeError(f"'float' object cannot be interpreted as an integer")
    v = operator.index(x)
    if not _INT_MIN <= v <= _INT_MAX:
        raise OverflowError("signed integer is greater than maximum" if v > 0 else "signed integer is less than minimum")
    return v


_SPACE_SETS: dict = {}


def _space_letters(letter_bytes: int, signed_bytes: bool) -> np.ndarray:
    """The package's one definition of white space: every letter value of the given width (as stored) for which libc
    iswspace() is true under the current LC_CTYPE (acb_space_letters), sorted -- the skip set of the white-space scans.
    signed_bytes: 1-byte letters are widened through a signed char first, as the reference's bytes build does
    (src/utils.c:199-202).  Cached per width, signedness and locale."""
    key = (letter_bytes, bool(signed_bytes), locale.setlocale(locale.LC_CTYPE))
    s = _SPACE_SETS.get(key)
    if s is None:
        lib, n, cap = N.lib(), ctypes.c_int64(0), 64
        while True:
            out = np.empty(cap, dtype=np.uint32)
            rc = lib.acb_space_letters(letter_bytes, int(bool(signed_bytes)), N.ptr(out), cap, ctypes.byref(n))
            if rc != N.ACB_EOVERFLOW:
                break
            cap = int(n.value)
        N.check(rc)
        s = out[:n.value].copy()
        s.flags.writeable = False
        _SPACE_SETS[key] = s
    return s


def _space_mask(letters: np.ndarray, bytes_flavour: bool) -> np.ndarray:
    """iswspace() of every letter, as the reference evaluates it (src/AutomatonSearchIter.c:270-274).
    The bytes flavour widens through a signed char first (src/utils.c:199-202)."""
    if letters.size == 0:
        return np.zeros(0, dtype=bool)
    w = letters.dtype.itemsize
    return np.isin(letters, _space_letters(w, bytes_flavour and w == 1))


_WORD_LETTERS_BYTES = b"0123456789ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz_"
_ASCII_LOWER = {c: c + 0x20 for c in range(0x41, 0x5B)}


def _ascii_fold(key):
    """A key with its 26 ASCII capitals made small and nothing else (bytes.lower() touches ASCII only; str.lower() would
    fold every letter, so str keys are translated)."""
    return key.lower() if isinstance(key, bytes) else key.translate(_ASCII_LOWER)


# the case folds of the batch methods, as a folded table records them (acb_table's fold): ascii_case_insensitive folds
# A-Z only (acb_table_upload_folded), case_insensitive folds through _unicode_fold_map (acb_table_upload_folded_map)
_FOLD_NONE, _FOLD_ASCII, _FOLD_UNICODE = 0, 1, 2


def _sfold(ch: str) -> str:
    """Unicode simple case folding of one letter: its casefold() when that is one letter, else its lower() when that is
    one letter, else itself"""
    f = ch.casefold()
    if len(f) == 1:
        return f
    f = ch.lower()
    return f if len(f) == 1 else ch


@functools.lru_cache(maxsize=None)
def _unicode_fold_map() -> Tuple[np.ndarray, np.ndarray]:
    """The fold of case_insensitive as (from, to): two sorted uint32 arrays of every code point that changes and the
    one it folds to.  Letters with equal _sfold (Unicode simple case folding) match each other, and each such class
    folds to its lowest code point, so every latin-1 letter folds into latin-1 (µ stays µ; Μ and μ fold to it) and the
    map restricted to from < 256 is the fold of 1-byte letters.  One letter maps to one letter: ß and ss, or ﬁ and fi,
    stay apart, and ΐ stays itself.  No Turkic rule: ı and İ match neither i nor I.  No normalisation: é and e + U+0301
    stay apart.  Surrogates and letter values above U+10FFFF fold to themselves.  The classes follow the Unicode version
    of the running Python's unicodedata (unicodedata.unidata_version).  About 1.1 M calls: built on first use, once
    per process."""
    classes: dict = {}
    for c in range(0x110000):
        classes.setdefault(_sfold(chr(c)), []).append(c)
    pairs = sorted((c, members[0]) for members in classes.values() if len(members) > 1 for c in members[1:])
    frm = np.array([a for a, _ in pairs], dtype=np.uint32)
    to = np.array([b for _, b in pairs], dtype=np.uint32)
    frm.flags.writeable = False
    to.flags.writeable = False
    return frm, to


@functools.lru_cache(maxsize=None)
def _unicode_fold_table() -> dict:
    """_unicode_fold_map as a str.translate table"""
    frm, to = _unicode_fold_map()
    return dict(zip(frm.tolist(), to.tolist()))


def _fold_key(key, kind: int):
    """A key folded as a table of fold kind _FOLD_ASCII or _FOLD_UNICODE folds its text"""
    return _ascii_fold(key) if kind == _FOLD_ASCII else key.translate(_unicode_fold_table())


class _FoldCore(NamedTuple):
    """The folded automaton of one letter width (Automaton._fold_host): its host trie, which holds each folded key under
    its group's representative (the lowest id of the keys that fold to it), and the alias lists of acb_table_upload_folded
    -- alias_ids[alias_ptr[k]:alias_ptr[k + 1]] are the other ids of representative k's group, ascending."""
    trie: Any
    alias_ptr: np.ndarray
    alias_ids: np.ndarray


@functools.lru_cache(maxsize=None)
def _default_word_mask(flavour: str) -> np.ndarray:
    """The default word letters: re's \\w -- [0-9A-Za-z_] over the 256 byte values for the bytes flavour, isalnum() or
    "_" over every code point for the unicode flavour (about 1.1 M calls: built on first use, once per process)."""
    if flavour == "bytes":
        m = np.zeros(256, dtype=bool)
        m[np.frombuffer(_WORD_LETTERS_BYTES, dtype=np.uint8)] = True
    else:
        m = np.fromiter((chr(c).isalnum() for c in range(0x110000)), dtype=bool, count=0x110000)
        m[ord("_")] = True
    m.flags.writeable = False
    return m


@functools.lru_cache(maxsize=64)
def _word_bits(words: tuple, width: int) -> Tuple[np.ndarray, int]:
    """(uint32 bitmap, n_bits) of a word set (Automaton._words) for letters of `width` bytes as a batch stores them: 1
    for the bytes flavour and for the unicode flavour's latin-1 batches (the first 256 code points), 4 otherwise.
    n_bits is one past the largest word letter, so a set without letters has no bitmap at all."""
    flavour, letters = words
    size = 256 if width == 1 else 0x110000
    if letters is None:
        mask = _default_word_mask(flavour)[:size]
    else:
        v = np.frombuffer(letters, dtype=np.uint8) if flavour == "bytes" else \
            np.fromiter(map(ord, letters), dtype=np.int64, count=len(letters))
        mask = np.zeros(size, dtype=bool)
        mask[v[v < size]] = True
    set_bits = np.flatnonzero(mask)
    n_bits = int(set_bits[-1]) + 1 if set_bits.size else 0
    packed = np.zeros(-(-n_bits // 32) * 4, dtype=np.uint8)
    packed[:-(-n_bits // 8)] = np.packbits(mask[:n_bits], bitorder="little")
    bits = packed.view("<u4")
    bits.flags.writeable = False
    return bits, n_bits


@functools.lru_cache(maxsize=64)
def _word_bits_device(words: tuple, width: int, device: int):
    """_word_bits on a CUDA device: (int32 CUDA tensor, n_bits), uploaded once per device, width and word set"""
    import torch
    bits, n_bits = _word_bits(words, width)
    return torch.from_numpy(bits.view(np.int32).copy()).to(f"cuda:{device}"), n_bits


class _PinnedRecords:
    """Owner of one pinned record buffer taken from the library (acb_take_records): exposes it to numpy through
    the array interface, gives it back (acb_release_records) when the last view is garbage collected."""
    __slots__ = ("_lib", "_ptr", "_cap", "__array_interface__")

    def __init__(self, lib, ptr: int, n: int, cap: int):
        self._lib, self._ptr, self._cap = lib, ptr, cap
        self.__array_interface__ = {"version": 3, "shape": (n,), "typestr": "|V12", "descr": N.MATCH_DTYPE.descr,
                                    "data": (ptr, False)}

    def __del__(self):
        try:
            self._lib.acb_release_records(self._ptr, self._cap)
        except Exception:                                   # interpreter shutdown
            pass


class Matches:
    """Result of a batch search: parallel int32 arrays in the reference's order
    (hay_id, then end_index ascending, then longest key first).  Its values are those of the key set at call time:
    later changes of the automaton do not reach them (Automaton._result_values)."""

    __slots__ = ("hay_id", "end_index", "key_id", "_values")

    def __init__(self, rec: np.ndarray, values: list):
        self.hay_id = rec["hay_id"]
        self.end_index = rec["end_index"]
        self.key_id = rec["key_id"]
        self._values = values

    def __len__(self):
        return len(self.hay_id)

    def values(self) -> list:
        v = self._values
        return [v[k] for k in self.key_id.tolist()]

    def __iter__(self):
        v = self._values
        return iter([(h, e, v[k]) for h, e, k in zip(self.hay_id.tolist(), self.end_index.tolist(), self.key_id.tolist())])

    def per_haystack(self, n_hay: int) -> List[List[Tuple[int, Any]]]:
        """[[(end_index, value), ...] for each haystack] -- what looping iter() would give."""
        out: List[List[Tuple[int, Any]]] = [[] for _ in range(n_hay)]
        v = self._values
        for h, e, k in zip(self.hay_id.tolist(), self.end_index.tolist(), self.key_id.tolist()):
            out[h].append((e, v[k]))
        return out


class Automaton:
    """Drop-in for ``ahocorasick.Automaton`` (src/Automaton.c:96-181 constructor)."""

    _UNICODE = True           # flavour; the bytes flavour subclass overrides it
    _long_state_out = 0       # state the last iter_long chunk ended in (acb_table_get_long_state), see AutomatonSearchIterLong

    # ------------------------------------------------------------------ construction
    def __init__(self, *args):
        store, key_type = STORE_ANY, KEY_STRING
        # src/Automaton.c:150-173: "ii" or "i"; anything else silently keeps the defaults
        if len(args) == 2 and all(isinstance(a, int) for a in args):
            store, key_type = args
            self._check_store(store)
            self._check_key_type(key_type)
        elif len(args) == 1 and isinstance(args[0], int):
            store = args[0]
            self._check_store(store)
        self._lib = N.lib()
        self._gpu_lock = threading.RLock()      # see _locked
        self._trie = None
        self._table = None
        self._narrow_trie = None
        self._narrow_table = None
        self._fold_cores = {}
        self._fold_tables = {}
        self._configure(store, key_type)
        if len(args) == 7:                # what __reduce__ of the reference produces, src/Automaton.c:106-147
            from . import serialize
            serialize.from_reduce_args(self, args)

    def _configure(self, store, key_type):
        """(re)start as an empty automaton of the given store / key type"""
        self._drop_table()
        if self._trie:
            self._lib.acb_trie_free(self._trie)
            self._trie = None
        self._store = store
        self._key_type = key_type
        self._L = self._letter_bytes()
        self._trie = self._lib.acb_trie_new(self._L)
        if not self._trie:
            raise MemoryError(N.last_error())
        self._key_ids: dict = {}          # key object -> key_id
        self._key_objs: list = []         # key_id -> key object (None once removed)
        self._values: list = []           # key_id -> value
        self._values_shared = False       # a result reads _values later: copy it before changing an entry (_own_values)
        self._version = 0
        self._table = None                # acb_table* (device), created lazily
        self._table_device = None
        # unicode flavour only: a second, 1-byte-per-letter automaton over the keys that are pure latin-1,
        # built lazily and used whenever a haystack is latin-1 too (4x fewer bytes to move and scan)
        self._narrow_trie = None
        self._narrow_table = None
        self._narrow_device = None
        self._narrow_empty = False
        # case folding: per (fold kind, narrow) the folded automaton (_FoldCore, or None without a key) and its table as
        # (acb_table*, device), built lazily
        self._fold_cores: dict = {}
        self._fold_tables: dict = {}
        self._match_cap = 0

    @staticmethod
    def _check_store(store):
        if store not in (STORE_INTS, STORE_LENGTH, STORE_ANY):
            raise ValueError("store value must be one of ahocorasick.STORE_LENGTH, STORE_INTS or STORE_ANY")

    @staticmethod
    def _check_key_type(key_type):
        if key_type not in (KEY_STRING, KEY_SEQUENCE):
            raise ValueError("key_type must have value KEY_STRING or KEY_SEQUENCE")

    def _letter_bytes(self) -> int:
        if self._key_type == KEY_SEQUENCE:
            return 4 if self._UNICODE else 2      # TRIE_LETTER_TYPE, src/common.h:51-67
        return 4 if self._UNICODE else 1

    def __del__(self):
        try:
            self._drop_table()
            if self._trie:
                self._lib.acb_trie_free(self._trie)
                self._trie = None
        except Exception:
            pass

    # ------------------------------------------------------------------ marshalling (src/utils.c:145-289)
    def _hay_letters(self, obj, required: bool = False) -> np.ndarray:
        """haystack -> letters; latin-1 `str` haystacks of the unicode flavour come back as uint8 (narrow path)."""
        if self._uses_narrow() and isinstance(obj, str):
            try:
                return np.frombuffer(obj.encode("latin-1"), dtype=np.uint8)
            except UnicodeEncodeError:
                pass
        return self._letters(obj, required)

    def _letters(self, obj, required: bool = False) -> np.ndarray:
        """key / haystack object -> array of letters (dtype by letter width)."""
        if self._key_type == KEY_SEQUENCE:
            if not isinstance(obj, tuple):
                raise TypeError("tuple required" if required else "argument is not a supported sequence type")
            hi = 2 ** 32 - 1 if self._UNICODE else 65535
            out = np.empty(len(obj), dtype=_LETTER_DTYPE[self._L])
            for i, item in enumerate(obj):
                try:
                    v = operator.index(item)
                except TypeError:
                    raise ValueError(f"item #{i} is not a number") from None
                if v < 0 or v > hi:
                    raise ValueError(f"item #{i}: value {v} outside range [0..{hi}]")
                out[i] = v
            return out
        if self._UNICODE:
            if not isinstance(obj, str):
                raise TypeError("string required" if required else "string expected")
            return np.frombuffer(obj.encode("utf-32-le", "surrogatepass"), dtype="<u4")
        if not isinstance(obj, bytes):
            raise TypeError("bytes required" if required else "bytes expected")
        return np.frombuffer(obj, dtype=np.uint8)

    def _raw_key(self, key):
        """key object -> (its letters as bytes, number of letters), without the numpy detour for plain string
        keys: the dict-like methods are called once per key, not once per batch"""
        if self._key_type == KEY_STRING:
            if self._UNICODE:
                if not isinstance(key, str):
                    raise TypeError("string expected")
                raw = key.encode("utf-32-le", "surrogatepass")
                return raw, len(raw) >> 2
            if not isinstance(key, bytes):
                raise TypeError("bytes expected")
            return key, len(key)
        letters = self._letters(key)
        return letters.tobytes(), len(letters)

    def _hashable(self, key):
        return key

    # ------------------------------------------------------------------ dict-like part (host trie)
    @property
    def kind(self) -> int:
        return self._lib.acb_trie_kind(self._trie)

    @property
    def store(self) -> int:
        return self._store

    def __len__(self):
        return self._lib.acb_trie_count(self._trie)

    @_locked
    def add_word(self, *args) -> bool:
        """src/Automaton.c:201-300."""
        if not args:
            raise TypeError("add_word() requires a key")      # PyTuple_GetItem -> IndexError in the reference
        key = args[0]
        raw, n = self._raw_key(key)
        if self._store == STORE_ANY:
            if len(args) < 2:
                raise ValueError("A value object is required as second argument.")
            value = args[1]
        elif self._store == STORE_INTS:
            if len(args) >= 2:
                v = args[1]
                if not isinstance(v, (int, float, np.integer)) and not hasattr(v, "__index__"):
                    raise TypeError("An integer value is required as second argument.")
                try:
                    iv = operator.index(v) if not isinstance(v, float) else None
                except TypeError:
                    iv = None
                if iv is None:
                    raise TypeError("'float' object cannot be interpreted as an integer")
                if not -(2 ** 63) <= iv < 2 ** 63:
                    raise ValueError("Python int too large to convert to C ssize_t")
                value = _to_c_int(iv)
            else:
                value = _to_c_int(len(self) + 1)               # :238-243 default
        else:
            value = n                                           # STORE_LENGTH :245-247
        if n == 0:
            return False                                        # :257,295
        hk = self._hashable(key)
        kid = self._key_ids.get(hk)
        new_id = len(self._values) if kid is None else kid
        prev = ctypes.c_int32(-1)
        N.check(self._lib.acb_trie_add_word(self._trie, raw, len(raw), new_id, ctypes.byref(prev)))
        self._drop_table()                                      # kind is TRIE again (src/trie.c:60)
        if kid is None:
            self._key_ids[hk] = new_id
            self._key_objs.append(key)
            self._values.append(value)
            self._version += 1                                  # :283-284
            return True
        self._own_values()
        self._values[kid] = value                               # replaced, version unchanged (A10)
        return False

    def _lookup(self, key):
        raw, _ = self._raw_key(key)
        kid = ctypes.c_int32(-1)
        pre = ctypes.c_int32(0)
        N.check(self._lib.acb_trie_find(self._trie, raw, len(raw), ctypes.byref(kid), ctypes.byref(pre)))
        return kid.value, bool(pre.value)

    def exists(self, key) -> bool:
        return self._lookup(key)[0] >= 0

    __contains__ = exists

    def match(self, key) -> bool:
        if self.kind == EMPTY:
            self._raw_key(key)
            return False
        return self._lookup(key)[1]

    def longest_prefix(self, key) -> int:
        raw, _ = self._raw_key(key)
        return int(self._lib.acb_trie_longest_prefix(self._trie, raw, len(raw)))

    _MISSING = object()

    def get(self, *args):
        if not 1 <= len(args) <= 2:
            raise TypeError(f"get() takes one or two arguments ({len(args)} given)")
        kid, _ = self._lookup(args[0])
        if kid >= 0:
            return self._values[kid]
        if len(args) == 2:
            return args[1]
        raise KeyError(args[0])

    def _remove(self, key):
        raw, n = self._raw_key(key)
        if n == 0:
            return None
        kid = ctypes.c_int32(-1)
        N.check(self._lib.acb_trie_remove_word(self._trie, raw, len(raw), ctypes.byref(kid)))
        if kid.value < 0:
            return None
        k = kid.value
        value = self._values[k]
        self._key_ids.pop(self._hashable(self._key_objs[k]), None)
        self._key_objs[k] = None
        self._own_values()
        self._values[k] = None
        self._version += 1
        self._drop_table()
        return (value,)

    @_locked
    def remove_word(self, key) -> bool:
        return self._remove(key) is not None

    @_locked
    def pop(self, key):
        r = self._remove(key)
        if r is None:
            raise KeyError(key)
        return r[0]

    @_locked
    def clear(self) -> None:
        N.check(self._lib.acb_trie_clear(self._trie))
        self._key_ids.clear()
        self._key_objs = []
        self._values = []
        self._values_shared = False
        self._version += 1
        self._drop_table()

    def _result_values(self):
        """_values for a result that reads them after the call (Matches), taken under the lock of the scan: from then on
        the list is copied before an entry of it changes (_own_values), so the result keeps the values of the key set it
        was computed on.  Adding keys appends to the list and needs no copy."""
        self._values_shared = True
        return self._values

    def _own_values(self):
        """before an entry of _values changes in place: a fresh copy of the list when a result holds it"""
        if self._values_shared:
            self._values = list(self._values)
            self._values_shared = False

    # keys / values / items (src/AutomatonItemsIter.c) -- host enumeration; keys_batch & co. run on the GPU
    def _select_args(self, args):
        """(prefix or None, wildcard letter value or None, how) of keys / values / items, checked in this order"""
        prefix = None
        wildcard = None
        how = MATCH_EXACT_LENGTH
        if len(args) >= 1 and args[0] is not None:
            prefix = args[0]
            self._letters(prefix)
        if len(args) >= 2 and args[1] is not None:
            wl = self._letters(args[1])
            if len(wl) != 1:
                raise ValueError("Wildcard must be a single character.")
            wildcard = int(wl[0])
        if len(args) >= 3:
            how = args[2]
            if how not in (MATCH_EXACT_LENGTH, MATCH_AT_MOST_PREFIX, MATCH_AT_LEAST_PREFIX):
                raise ValueError("The optional how third argument must be one of: "
                                 "MATCH_EXACT_LENGTH, MATCH_AT_LEAST_PREFIX or MATCH_AT_LEAST_PREFIX")
        return prefix, wildcard, how

    def _select(self, args):
        prefix, w, how = self._select_args(args)
        version = self._version
        # the reference's order: a pre-order walk of the trie that takes a node's youngest child first
        # (src/AutomatonItemsIter.c:125-288); the host trie knows it (acb_trie_key_order)
        n_live = len(self)
        order = np.empty(max(n_live, 1), dtype=np.int32)
        got = ctypes.c_int64(0)
        N.check(self._lib.acb_trie_key_order(self._trie, N.ptr(order), n_live, ctypes.byref(got)))
        ko, vals = self._key_objs, self._values
        live = [(ko[i], vals[i]) for i in order[:got.value].tolist()]
        if prefix is None:
            sel = live
        else:
            p = list(self._letters(prefix).tolist())
            sel = []
            for k, v in live:
                kl = self._letters(k).tolist()
                if w is None:
                    ok = kl[:len(p)] == p
                else:
                    if how == MATCH_EXACT_LENGTH and len(kl) != len(p):
                        continue
                    if how == MATCH_AT_MOST_PREFIX and len(kl) > len(p):
                        continue
                    if how == MATCH_AT_LEAST_PREFIX and len(kl) < len(p):
                        continue
                    m = min(len(kl), len(p))
                    ok = all(p[i] == w or p[i] == kl[i] for i in range(m))
                if ok:
                    sel.append((k, v))
        return version, sel

    def _guarded(self, version, seq):
        for x in seq:
            if version != self._version:
                raise ValueError("underlaying automaton has changed, iterator is not valid anymore")
            yield x

    def keys(self, *args):
        ver, sel = self._select(args)
        return self._guarded(ver, [k for k, _ in sel])

    def values(self, *args):
        ver, sel = self._select(args)
        return self._guarded(ver, [v for _, v in sel])

    def items(self, *args):
        ver, sel = self._select(args)
        return self._guarded(ver, sel)

    def __iter__(self):
        return self.keys()

    def get_stats(self) -> dict:
        """src/Automaton.c:1044-1097.  nodes / links / words / longest_word describe the trie of LETTERS exactly as
        the reference counts them (one node per letter, also for 2- and 4-byte letters; longest_word is the depth
        of the live trie, so unlike the attribute behind `save` it shrinks when the longest key is removed);
        sizeof_node / total_size are this implementation's own host memory: 32-byte arena nodes, one per BYTE of
        a letter, plus the edge table that indexes wide fan-outs (acb_trie_host_bytes)."""
        byte_nodes = int(self._lib.acb_trie_nodes(self._trie))
        nodes, links = byte_nodes, int(self._lib.acb_trie_links(self._trie))
        if self._L > 1 and byte_nodes:
            need, n = ctypes.c_int64(0), ctypes.c_int64(0)
            N.check(self._lib.acb_trie_export_nodes(self._trie, 4 if self._L == 4 else 2, None, 0, None, 0,
                                                    ctypes.byref(need), ctypes.byref(n), None, None, 0))
            nodes, links = n.value, max(n.value - 1, 0)
        longest = max((len(k) for k in self._key_objs if k is not None), default=0)
        node_bytes = 32                                   # arena Node in csrc/acb_host.cpp
        return dict(nodes_count=nodes, words_count=len(self), longest_word=longest, links_count=links,
                    sizeof_node=node_bytes, total_size=int(self._lib.acb_trie_host_bytes(self._trie)))

    def __sizeof__(self):
        return object.__sizeof__(self) + self.get_stats()["total_size"]

    def __reduce__(self):
        """src/Automaton_pickle.c:199-262: (Automaton, (bytes_list, kind, store, key_type, count, longest_word,
        values)), or (Automaton, ()) without keys.  The argument tuple is the reference's own format -- the
        reference's constructor accepts it and this constructor accepts the reference's (serialize.py).  An
        instance of the flavour that is not the package default is rebuilt through _rebuild, because both flavour
        classes answer to the name `Automaton`."""
        from . import serialize
        import pyahocorasick_b200 as pkg
        args = serialize.reduce_args(self)
        if type(self) is getattr(pkg, "Automaton", None):
            return (type(self), args)
        return (_rebuild, (type(self)._UNICODE, args))

    def save(self, *args):
        """save(path[, serializer]) in the reference's file format (src/custompickle/save/automaton_save.c)."""
        from . import serialize
        serialize.save(self, *args)

    # ------------------------------------------------------------------ automaton
    @_locked
    def make_automaton(self):
        """src/Automaton.c:560-649 -> None when built, False when there was nothing to do."""
        built = ctypes.c_int32(0)
        N.check(self._lib.acb_trie_make_automaton(self._trie, ctypes.byref(built)))
        if not built.value:
            return False
        self._version += 1                                 # :640
        self._drop_table()
        return None

    @_locked
    def _make_automaton_cached(self, cache_path: Optional[str] = None):
        """make_automaton() for an automaton that comes out of a file or a pickle (SURVEY 8(f) #2): the reference's
        files carry the failure links, so a loaded automaton is searchable at once; here everything make_automaton
        derives from the key set (goto / fail / outputs / gram filter / anchors) is cached in a file keyed by a content
        hash of the key set -- `cache_path` (load() passes `<file>.acb200`), else `$ACB200_CACHE_DIR/<hash>.acb200`
        when that variable names a directory.  A hit installs the tables without BFS, flatten or filter construction;
        a miss builds them and writes the cache (best effort: an unwritable place is not an error)."""
        if self.kind != TRIE:
            return self.make_automaton()
        if cache_path is None:
            d = os.environ.get("ACB200_CACHE_DIR")
            if d and os.path.isdir(d):
                cache_path = os.path.join(d, "%016x.acb200" % int(self._lib.acb_trie_content_hash(self._trie)))
        if cache_path is not None and os.path.exists(cache_path):
            try:
                blob = np.fromfile(cache_path, dtype=np.uint8)
                if self._lib.acb_trie_flat_load(self._trie, N.ptr(blob), int(blob.size)) == N.ACB_OK:
                    self._version += 1
                    self._drop_table()
                    return None
            except OSError:
                pass
        r = self.make_automaton()
        if cache_path is not None and self.kind == AHOCORASICK:
            try:
                need = ctypes.c_int64(0)
                N.check(self._lib.acb_trie_flat_save(self._trie, None, 0, ctypes.byref(need)))
                blob = np.empty(need.value, dtype=np.uint8)
                N.check(self._lib.acb_trie_flat_save(self._trie, N.ptr(blob), need.value, ctypes.byref(need)))
                tmp = cache_path + ".tmp%d" % os.getpid()
                blob.tofile(tmp)
                os.replace(tmp, cache_path)
            except (OSError, N.NativeError):
                pass
        return r

    @_locked
    def _drop_table(self):
        if self._table is not None:
            self._lib.acb_table_free(self._table)
            self._table = None
        if self._narrow_table is not None:
            self._lib.acb_table_free(self._narrow_table)
            self._narrow_table = None
        if self._narrow_trie is not None:
            self._lib.acb_trie_free(self._narrow_trie)
            self._narrow_trie = None
        self._narrow_empty = False
        for tb, _ in self._fold_tables.values():
            self._lib.acb_table_free(tb)
        self._fold_tables = {}
        for core in self._fold_cores.values():
            if core is not None:
                self._lib.acb_trie_free(core.trie)
        self._fold_cores = {}

    def _uses_narrow(self) -> bool:
        return self._UNICODE and self._key_type == KEY_STRING

    @_locked
    def _narrow_host(self):
        """host trie of the latin-1 automaton (built lazily), or None when no key is pure latin-1."""
        if self._narrow_empty:
            return None
        if self._narrow_trie is None:
            t = self._lib.acb_trie_new(1)
            if not t:
                raise MemoryError(N.last_error())
            n = 0
            for kid, key in enumerate(self._key_objs):
                if key is None:
                    continue
                try:
                    raw = key.encode("latin-1")
                except UnicodeEncodeError:
                    continue                                    # cannot occur in a latin-1 haystack
                N.check(self._lib.acb_trie_add_word(t, raw, len(raw), kid, None))
                n += 1
            if n == 0:
                self._lib.acb_trie_free(t)
                self._narrow_empty = True
                return None
            built = ctypes.c_int32(0)
            N.check(self._lib.acb_trie_make_automaton(t, ctypes.byref(built)))
            self._narrow_trie = t
        return self._narrow_trie

    @_locked
    def _ensure_narrow(self, device: Optional[int]):
        """(trie, table) of the latin-1 automaton, or None when no key is pure latin-1."""
        if self._narrow_host() is None:
            return None
        if device is None:
            device = _default_device()
        if self._narrow_table is None or self._narrow_device != device:
            if self._narrow_table is not None:
                self._lib.acb_table_free(self._narrow_table)
                self._narrow_table = None
            tb = ctypes.c_void_p()
            N.check(self._lib.acb_table_upload(self._narrow_trie, device, ctypes.byref(tb)))
            self._narrow_table = tb
            self._narrow_device = device
        return self._narrow_trie, self._narrow_table

    @_locked
    def _ensure_table(self, device: Optional[int] = None):
        if device is None:
            device = _default_device()
        if self._table is not None and self._table_device == device:
            return self._table
        self._drop_table()
        tb = ctypes.c_void_p()
        N.check(self._lib.acb_table_upload(self._trie, device, ctypes.byref(tb)))
        self._table = tb
        self._table_device = device
        return tb

    @_locked
    def _fold_host(self, narrow: bool, kind: int = _FOLD_ASCII) -> Optional[_FoldCore]:
        """The folded automaton of a fold kind (_FOLD_ASCII or _FOLD_UNICODE) and a batch's letter width (narrow: the
        keys whose folded text is latin-1, at 1 byte per letter), built lazily; None when it has no key.  Keys are added in
        ascending id, and a key whose folded text is already there is not added but listed as an alias of the id that
        holds it, so that id is the lowest of its group."""
        if (kind, narrow) in self._fold_cores:
            return self._fold_cores[(kind, narrow)]
        t = self._lib.acb_trie_new(1 if narrow else self._L)
        if not t:
            raise MemoryError(N.last_error())
        reps: dict = {}
        aliases: dict = {}
        for kid, key in enumerate(self._key_objs):
            if key is None:
                continue
            folded = _fold_key(key, kind)
            if narrow:
                try:
                    raw = folded.encode("latin-1")
                except UnicodeEncodeError:
                    continue                                    # cannot occur in a latin-1 haystack
            else:
                raw, _ = self._raw_key(folded)
            rep = reps.setdefault(raw, kid)
            if rep != kid:
                aliases.setdefault(rep, []).append(kid)
                continue
            N.check(self._lib.acb_trie_add_word(t, raw, len(raw), kid, None))
        if not reps:
            self._lib.acb_trie_free(t)
            self._fold_cores[(kind, narrow)] = None
            return None
        built = ctypes.c_int32(0)
        N.check(self._lib.acb_trie_make_automaton(t, ctypes.byref(built)))
        alias_ptr = np.zeros(max(reps.values()) + 2, dtype=np.int32)
        for rep, ids in aliases.items():
            alias_ptr[rep + 1] = len(ids)
        np.cumsum(alias_ptr, out=alias_ptr)
        alias_ids = np.array([k for rep in sorted(aliases) for k in aliases[rep]], dtype=np.int32)
        core = self._fold_cores[(kind, narrow)] = _FoldCore(t, alias_ptr, alias_ids)
        return core

    @_locked
    def _ensure_folded(self, device: Optional[int], narrow: bool, kind: int = _FOLD_ASCII):
        """The folded table of a fold kind and a batch's letter width on `device` (acb_table_upload_folded, or
        acb_table_upload_folded_map with _unicode_fold_map); None when it has no key."""
        core = self._fold_host(narrow, kind)
        if core is None:
            return None
        if device is None:
            device = _default_device()
        have = self._fold_tables.get((kind, narrow))
        if have is not None and have[1] == device:
            return have[0]
        if have is not None:
            self._lib.acb_table_free(have[0])
            del self._fold_tables[(kind, narrow)]
        tb = ctypes.c_void_p()
        n = len(core.alias_ids)
        aliases = (core.trie, device, N.ptr(core.alias_ptr) if n else None, N.ptr(core.alias_ids) if n else None, n)
        if kind == _FOLD_ASCII:
            N.check(self._lib.acb_table_upload_folded(*aliases, ctypes.byref(tb)))
        else:
            frm, to = _unicode_fold_map()
            if narrow:
                frm, to = np.ascontiguousarray(frm[frm < 256]), np.ascontiguousarray(to[frm < 256])
            N.check(self._lib.acb_table_upload_folded_map(*aliases, N.ptr(frm), N.ptr(to), len(frm), ctypes.byref(tb)))
        self._fold_tables[(kind, narrow)] = (tb, device)
        return tb

    def _table_for(self, device: Optional[int], narrow: bool, fold: int = _FOLD_NONE):
        """The table a batch runs on: the latin-1 one for a narrow batch, else the full one; with a fold kind, the folded
        table of that kind and width.  None when the batch is narrow and no key is latin-1: then nothing matches."""
        if fold:
            return self._ensure_folded(device, narrow, fold)
        if not narrow:
            return self._ensure_table(device)
        core = self._ensure_narrow(device)
        return None if core is None else core[1]

    def _has_aliases(self, narrow: bool, kind: int = _FOLD_ASCII) -> bool:
        """the folded key set of this kind and width has case variants (an alias expansion follows the find_all scans)"""
        core = self._fold_host(narrow, kind)
        return core is not None and len(core.alias_ids) > 0

    def _fold_arg(self, ascii_case_insensitive, algo: str = "auto", ignore_white_space: bool = False,
                  case_insensitive: bool = False) -> int:
        """The fold kind that the ascii_case_insensitive and case_insensitive arguments of the batch methods ask for
        (_FOLD_NONE, _FOLD_ASCII or _FOLD_UNICODE), checked against the others"""
        if not ascii_case_insensitive and not case_insensitive:
            return _FOLD_NONE
        name = "case_insensitive" if case_insensitive else "ascii_case_insensitive"
        if self._key_type == KEY_SEQUENCE:
            raise ValueError(f"{name} needs text: KEY_SEQUENCE letters are integers, not letters")
        if ascii_case_insensitive and case_insensitive:
            raise ValueError("case_insensitive and ascii_case_insensitive are two different folds: pass one of them")
        if case_insensitive and not self._UNICODE:
            raise ValueError("case_insensitive folds code points, and bytes have no known encoding: the bytes flavour "
                             "takes ascii_case_insensitive")
        if ignore_white_space:
            raise ValueError(f"{name} cannot be combined with ignore_white_space")
        if algo == "long":
            raise ValueError(f"{name} cannot be combined with algo='long'")
        return _FOLD_UNICODE if case_insensitive else _FOLD_ASCII

    @_locked
    def filter_shape(self) -> dict:
        """The prefilter the host chose for this key set (no table copies): gram length, probe stride, bitmap sizes
        and the placement flags -- ACB_FILTER_PAIR (2) means the scan runs on acb_pair_kernel, else acb_stream_kernel."""
        fv = N.FlatView()
        N.check(self._lib.acb_trie_flat_view(self._trie, ctypes.byref(fv)))
        return dict(gram_bytes=fv.gram_bytes, stride=fv.stride, log2_bits1=fv.log2_bits1, log2_bits2=fv.log2_bits2,
                    log2_bits3=fv.log2_bits3, log2_anchor_slots=fv.log2_anchor_slots, filter_flags=fv.filter_flags)

    @_locked
    def flat(self, narrow: bool = False) -> dict:
        """White-box view of the flattened automaton (numpy copies) -- used by tests and docs.
        narrow=True: the latin-1 automaton of a unicode-flavour Automaton (None if it has no latin-1 key)."""
        trie = self._trie
        if narrow:
            trie = self._narrow_host()
            if trie is None:
                return None
        return self._flat_view(trie)

    def _flat_view(self, trie) -> dict:
        """flat() of a host trie of this automaton (also the folded ones of _fold_host)"""
        fv = N.FlatView()
        N.check(self._lib.acb_trie_flat_view(trie, ctypes.byref(fv)))
        S, K = fv.n_states, fv.n_classes

        def arr(p, n, dt):
            if n == 0 or not p:                       # e.g. no outputs at all once every key has been removed
                return np.empty(0, dtype=dt)
            return np.ctypeslib.as_array(p, shape=(n,)).astype(dt, copy=True)
        n_out = int(np.ctypeslib.as_array(fv.out_ptr, shape=(S + 1,))[S])
        return dict(
            n_states=S, n_classes=K, n_keys=fv.n_keys, letter_bytes=fv.letter_bytes,
            min_key_bytes=fv.min_key_bytes, max_key_bytes=fv.max_key_bytes,
            byte_class=arr(fv.byte_class, 256, np.uint8), goto_cm=arr(fv.goto_cm, K * S, np.int32).reshape(K, S),
            fail=arr(fv.fail, S, np.int32), letter_fail=arr(fv.letter_fail, S, np.int32), key_of=arr(fv.key_of, S, np.int32), out_ptr=arr(fv.out_ptr, S + 1, np.int32),
            out_idx=arr(fv.out_idx, n_out, np.int32), key_len=arr(fv.key_len, fv.n_keys, np.int32),
            gram_bytes=fv.gram_bytes, stride=fv.stride, log2_bits1=fv.log2_bits1,
            log2_anchor_slots=fv.log2_anchor_slots, filter_flags=fv.filter_flags, log2_bits3=fv.log2_bits3,
            bitmap3=arr(fv.bitmap3, (1 << (fv.log2_bits3 - 5)) if fv.log2_bits3 else 1, np.uint32),
            log2_bits2=fv.log2_bits2,
            bitmap1=arr(fv.bitmap1, (1 << (fv.log2_bits1 - 5)) + ((1 << (fv.log2_bits2 - 5)) if fv.log2_bits2 else 0), np.uint32),
            anchors=arr(fv.anchors, 8 << fv.log2_anchor_slots, np.uint32).reshape(-1, 8))

    # ------------------------------------------------------------------ GPU scan plumbing
    @_locked
    def _scan_flat(self, flat: np.ndarray, offsets: Optional[np.ndarray], n_hay: int, stride_bytes: int,
                   algo: str = "auto", sort: bool = True, device: Optional[int] = None, narrow: bool = False,
                   long_state: Optional[int] = None, fold: int = _FOLD_NONE) -> np.ndarray:
        """flat uint8 buffer (+ int64 byte offsets or a fixed stride) -> sorted match records.
        narrow=True: the buffer holds 1-byte letters of a unicode-flavour automaton (latin-1 path).  fold: on the folded
        table, which folds the text and expands the aliases itself.
        long_state (algo "long", one haystack): the state the walk starts in; the state it ends in is left in
        self._long_state_out (iter_long streaming, acb_table_set_long_state / acb_table_get_long_state)."""
        lib, total = self._lib, int(flat.size)

        def scan(tb, cap, found_ref):
            if long_state is not None:
                N.check(lib.acb_table_set_long_state(tb, int(long_state)))      # one shot: again before a retry
            rc = lib.acb_scan_host(tb, N.ptr(flat) if total else None, total, N.ptr(offsets) if offsets is not None else None,
                                   n_hay, stride_bytes, None, cap, found_ref, N.ALGOS[algo], 1 if sort else 0)
            if rc == N.ACB_OK and long_state is not None:
                st = ctypes.c_int32(0)
                N.check(lib.acb_table_get_long_state(tb, ctypes.byref(st)))
                self._long_state_out = int(st.value)
            return rc
        return self._host_records(device, narrow, n_hay, scan, fold)

    def _record_room(self, n_hay: int) -> int:
        """The first guess of the records a batch of n_hay haystacks gives; _match_cap remembers the largest overflow."""
        return max(self._match_cap, 1 << 12, 2 * n_hay)

    def _host_records(self, device: Optional[int], narrow: bool, n_hay: int, call, fold: int = _FOLD_NONE) -> np.ndarray:
        """The records of one host-buffer call, which leaves them in its table's pinned buffer.  call(tb, cap, found_ref)
        makes the native call with room for cap records and returns its status.  On ACB_EOVERFLOW it runs once more with
        room for the exact count (+1024, kept in _match_cap); a second overflow raises.  The records are handed over
        without a copy (_take_records).  fold: on the folded table (_table_for)."""
        tb = self._table_for(device, narrow, fold)
        if tb is None:
            return np.empty(0, dtype=N.MATCH_DTYPE)
        return self._host_records_on(tb, n_hay, call)

    def _host_records_on(self, tb, n_hay: int, call) -> np.ndarray:
        """_host_records on the table tb"""
        found = ctypes.c_int64(0)
        rc = call(tb, self._record_room(n_hay), ctypes.byref(found))
        if rc == N.ACB_EOVERFLOW:
            self._match_cap = int(found.value) + 1024
            rc = call(tb, self._match_cap, ctypes.byref(found))
        N.check(rc)
        if not found.value:
            return np.empty(0, dtype=N.MATCH_DTYPE)
        return _take_records(self._lib, tb, found.value)

    def _device_scan(self, t, n_hay: int, call):
        """The records of one device call on torch's current stream, left on the device: (int32 [cap, 3] CUDA tensor,
        their number).  call(out, cap, cnt) makes the native call into out with its int64 count cnt, zeroed before each
        try.  When the count exceeds cap (nothing was committed), it runs once more with room for it (+1024, kept in
        _match_cap); a second overflow raises."""
        import torch
        cnt = torch.empty(1, dtype=torch.int64, device=t.device)
        cap = self._record_room(n_hay)
        for retry in (False, True):
            out = torch.empty((cap, 3), dtype=torch.int32, device=t.device)
            cnt.zero_()
            call(out, cap, cnt)
            found = int(cnt.item())
            if found <= cap:
                return out, found
            if retry:
                raise N.NativeError(f"{found} records after a retry with room for {cap}")
            cap = self._match_cap = found + 1024

    def _words(self, whole_words):
        """The whole_words argument of the batch methods, parsed once: None for False, else the word set as
        (flavour, letters) with letters None for the default set (see _word_bits)."""
        if whole_words is False:
            return None
        if self._key_type == KEY_SEQUENCE:
            raise ValueError("whole_words needs text: KEY_SEQUENCE letters are integers, not letters of words")
        flavour = "unicode" if self._UNICODE else "bytes"
        if whole_words is True:
            return (flavour, None)
        if isinstance(whole_words, (bytes, bytearray, str)):
            if isinstance(whole_words, str) != self._UNICODE:
                raise ValueError(f"whole_words of the {flavour} flavour is True or a {'str' if self._UNICODE else 'bytes'} "
                                 "of word letters")
            return (flavour, whole_words if isinstance(whole_words, str) else bytes(whole_words))
        raise TypeError("whole_words must be a bool, or the word letters as bytes (bytes flavour) or str (unicode flavour)")

    @_locked
    def _words_host(self, flat: np.ndarray, offsets: Optional[np.ndarray], n_hay: int, stride_bytes: int, algo: str, sort: bool,
                    device: Optional[int], narrow: bool, words: tuple, leftmost: bool, select: int = N.SELECT_LONGEST,
                    fold: int = _FOLD_NONE) -> np.ndarray:
        """acb_scan_host_words / acb_scan_host_leftmost_words (acb_scan_host_leftmost_kind for leftmost-first): upload,
        scan, keep the whole-word matches, then sort or select, copy back (_host_records)."""
        lib = self._lib
        bits, n_bits = _word_bits(words, 1 if narrow else self._L)
        args = (N.ptr(flat), int(flat.size), N.ptr(offsets) if offsets is not None else None, n_hay, stride_bytes,
                N.ptr(bits) if n_bits else None, n_bits, None)

        def scan(tb, cap, found_ref):
            if leftmost and select != N.SELECT_LONGEST:
                return lib.acb_scan_host_leftmost_kind(tb, select, *args, cap, found_ref, N.ALGOS[algo])
            if leftmost:
                return lib.acb_scan_host_leftmost_words(tb, *args, cap, found_ref, N.ALGOS[algo])
            return lib.acb_scan_host_words(tb, *args, cap, found_ref, N.ALGOS[algo], int(sort))
        return self._host_records(device, narrow, n_hay, scan, fold)

    def _filter_words_device(self, tb, t, n: int, stride: int, full, m: int, words: tuple, stream, offs=None, narrow: bool = False):
        """The whole-word records among the first m of the device buffer `full` (a scan of the aligned device batch t),
        on `stream`: (records [max(m, 1), 3] int32 CUDA tensor, their number).  Waits once, for that number.  offs: the
        batch's int64 CUDA byte offsets instead of rows of `stride` bytes; narrow: its letters are 1 byte each."""
        import torch
        bits, n_bits = _word_bits_device(words, 1 if narrow else self._L, t.device.index)
        out = torch.empty((max(m, 1), 3), dtype=torch.int32, device=t.device)
        cnt = torch.zeros(1, dtype=torch.int64, device=t.device)
        N.check(self._lib.acb_word_filter_device(tb, t.data_ptr(), t.numel(), None if offs is None else offs.data_ptr(), n, stride,
                                                 full.data_ptr(), m,
                                                 bits.data_ptr() if n_bits else None, n_bits, out.data_ptr(), m, cnt.data_ptr(),
                                                 stream))
        return out, int(cnt.item())

    @_locked
    def _scan_device_tensor(self, batch, algo: str, sort: bool, words: Optional[tuple] = None,
                            white_space: bool = False, fold: int = _FOLD_NONE) -> np.ndarray:
        """Batch already resident in HBM: a C-contiguous uint8 torch CUDA tensor [n, stride].  No host copy of
        the haystacks; the scan runs on torch's current stream, only the records come back.  words: keep the
        whole-word matches (_filter_words_device) before the sort.  white_space: the scan skips the white space
        (acb_scan_device_skip).  fold: on the folded table, with the aliases expanded after the word filter; the stable
        sort keeps each group's records in ascending id."""
        t = _aligned(batch.data)
        dev = _device_of(t)
        tb = self._table_for(dev, False, fold)
        skip = self._skip_set(False) if white_space else None
        with _on_device(dev) as stream:
            out, found = self._device_matches(tb, t, batch.n, batch.stride, algo, stream, words, skip)
            if fold and found and self._has_aliases(False, fold):
                out, found = self._expand_device(tb, t, batch.n, out, found, stream)
            return self._device_records(tb, out, found, batch.n, batch.stride // self._L, stream, sort)

    def _expand_device(self, tb, t, n: int, full, m: int, stream):
        """The first m records of the device buffer `full` with every alias of their key added (acb_expand_aliases_device),
        left on the device (_device_scan)."""
        def expand(out, cap, cnt):
            N.check(self._lib.acb_expand_aliases_device(tb, full.data_ptr(), m, out.data_ptr(), cap, cnt.data_ptr(), stream))
        return self._device_scan(t, n, expand)

    def _device_matches(self, tb, t, n: int, stride: int, algo: str, stream, words: Optional[tuple] = None,
                        skip: Optional[np.ndarray] = None, offs=None, narrow: bool = False):
        """Every match of the aligned device batch t, left on the device (_device_scan): (int32 [cap, 3] CUDA tensor,
        their number).  skip: the scan skips these letters; words: only the whole-word matches (_filter_words_device).
        offs, narrow: as for _filter_words_device."""
        lib = self._lib
        d_off = None if offs is None else offs.data_ptr()

        def scan(out, cap, cnt):
            args = (tb, t.data_ptr(), t.numel(), d_off, n, stride, out.data_ptr(), cap, cnt.data_ptr(), stream, N.ALGOS[algo])
            N.check(lib.acb_scan_device(*args) if skip is None else lib.acb_scan_device_skip(*args, N.ptr(skip), len(skip)))
        out, found = self._device_scan(t, n, scan)
        if words is not None:
            out, found = self._filter_words_device(tb, t, n, stride, out, found, words, stream, offs, narrow)
        return out, found

    def _device_records(self, tb, out, found: int, n_hay: int, max_letters: int, stream, sort: bool) -> np.ndarray:
        """The first `found` records of the device buffer `out`, sorted on the device (on the host when the sort key
        does not fit 64 bits), as numpy records."""
        sort_on_host = False
        if sort and found > 1:
            rc = self._lib.acb_sort_matches_device(tb, out.data_ptr(), found, n_hay, max_letters, stream)
            if rc == N.ACB_ERANGE:
                sort_on_host = True
            else:
                N.check(rc)
        rec = out[:found].cpu().numpy().view(N.MATCH_DTYPE).reshape(-1)
        if sort_on_host:
            kl = np.asarray(self.flat()["key_len"])
            rec = rec[np.lexsort((-kl[rec["key_id"]], rec["end_index"], rec["hay_id"]))]
        return rec

    def _skip_set(self, narrow: bool) -> np.ndarray:
        """The white-space letters of a batch, as its buffer stores them: 1-byte letters of a latin-1 batch (unicode
        flavour) or of the bytes flavour (widened through a signed char), 2-byte items of bytes-flavour sequences,
        4-byte letters otherwise."""
        if narrow:
            return _space_letters(1, False)
        return _space_letters(self._L, not self._UNICODE and self._key_type == KEY_STRING)

    @_locked
    def _scan_skip(self, batch, algo: str, sort: bool, device: Optional[int]) -> np.ndarray:
        """Every host scan with ignore_white_space: `batch`, a host batch as _batch_input lays it out -> records in
        original letters.  The white space is removed on the GPU (acb_scan_host_skip)."""
        lib = self._lib
        _, flat, offs, n, stride, narrow = batch
        skip = self._skip_set(narrow)

        def scan(tb, cap, found_ref):
            return lib.acb_scan_host_skip(tb, N.ptr(flat), int(flat.size), N.ptr(offs) if offs is not None else None, n,
                                          stride, None, cap, found_ref, N.ALGOS[algo], int(sort), N.ptr(skip), len(skip))
        return self._host_records(device, narrow, n, scan)

    def _device_batch_shape(self, t):
        """(n, stride_bytes) of a device batch: a C-contiguous uint8 torch CUDA tensor [n, stride]"""
        import torch
        if t.dtype != torch.uint8 or t.dim() != 2 or not t.is_contiguous():
            raise TypeError("device batches must be 2-D contiguous uint8 tensors [n_haystacks, stride_bytes]")
        n, stride = int(t.shape[0]), int(t.shape[1])
        if stride % self._L:
            raise ValueError("row length must be a multiple of the letter width")
        return n, stride

    def _scan_one(self, letters: np.ndarray, algo: str = "auto", long_state: Optional[int] = None) -> np.ndarray:
        narrow = self._uses_narrow() and letters.dtype == np.uint8 and algo != "long"
        if self._uses_narrow() and letters.dtype == np.uint8 and not narrow:
            letters = letters.astype("<u4")                  # iter_long never runs on the latin-1 automaton
        flat = np.ascontiguousarray(letters).view(np.uint8)
        if flat.size == 0:
            return np.empty(0, dtype=N.MATCH_DTYPE)
        return self._scan_flat(flat, None, 1, int(flat.size), algo=algo, narrow=narrow, long_state=long_state)

    def _require_automaton(self):
        if self.kind != AHOCORASICK:
            raise AttributeError("Not an Aho-Corasick automaton yet: call add_word to add some keys and call "
                                 "make_automaton to convert the trie to an automaton.")

    # ------------------------------------------------------------------ search API of the reference
    @_locked
    def iter(self, *args, **kwargs):
        """src/Automaton.c:875-966: iter(string, [start, [end]], ignore_white_space=False)."""
        self._require_automaton()
        names = ("string", "start", "end", "ignore_white_space")
        if len(args) > 4:
            raise TypeError(f"function takes at most 4 arguments ({len(args)} given)")
        vals = dict(zip(names, args))
        for k, v in kwargs.items():
            if k not in names:
                raise TypeError(f"'{k}' is an invalid keyword argument for this function")
            if k in vals:
                raise TypeError(f"argument for function given by name ('{k}') and position")
            vals[k] = v
        if "string" not in vals:
            raise TypeError("function missing required argument 'string' (pos 1)")
        start = _parse_c_int(vals.get("start", -1))
        end = _parse_c_int(vals.get("end", -1))
        iws = _parse_c_int(vals.get("ignore_white_space", -1)) == 1          # :897-899 (A6)
        letters = self._hay_letters(vals["string"], required=True)
        n = len(letters)
        if start == -1:
            start = 0                                                         # -1 = "not given" (A2)
        if end == -1:
            end = n
        # the reference does not validate the range (A1: out-of-bounds read); parity is defined for
        # 0 <= start <= end <= len, anything else is clamped
        start = min(max(start, 0), n)
        end = min(max(end, 0), n)
        return AutomatonSearchIter(self, letters, start, end, iws)

    def find_all(self, *args):
        """src/Automaton.c:652-719: find_all(string, callback, [start, [end]])."""
        if self.kind != AHOCORASICK:
            return None                                                        # :666-667 (A4)
        if len(args) < 1:
            raise IndexError("tuple index out of range")
        letters = self._hay_letters(args[0])
        if len(args) < 2:
            raise IndexError("tuple index out of range")
        callback = args[1]
        if not callable(callback):
            raise TypeError("The callback argument must be a callable such as a function.")
        start, end = _parse_start_end(args, 2, 3, 0, len(letters))
        if end > start:
            rec = self._scan_one(letters[start:end])
            values = self._values
            for e, k in zip(rec["end_index"].tolist(), rec["key_id"].tolist()):
                callback(e + start, values[k])
        return None

    @_locked
    def iter_long(self, *args):
        """src/Automaton.c:968-1040 + src/AutomatonSearchIterLong.c:89-153: iter_long(string, [start, [end]]) --
        longest, non-overlapping matches.  One GPU lane replays the reference's state machine per haystack."""
        if self.kind != AHOCORASICK:
            raise AttributeError("not an automaton yet; add some words and call make_automaton")
        if len(args) < 1:
            raise IndexError("tuple index out of range")
        letters = self._letters(args[0], required=True)      # never the latin-1 automaton: see find_all_batch
        start, end = _parse_start_end(args, 1, 2, 0, len(letters))
        return AutomatonSearchIterLong(self, letters, start, end)

    def find_long_batch(self, haystacks, *, sort: bool = True, device: Optional[int] = None, whole_words=False,
                        ascii_case_insensitive: bool = False, case_insensitive: bool = False, encoding: Optional[str] = None,
                        errors: str = "strict") -> "Matches":
        """iter_long() over a whole batch (same input forms and result type as find_all_batch).  whole_words,
        ascii_case_insensitive and case_insensitive are refused (ValueError): iter_long's walk picks its matches itself,
        so a filter after it has no clear meaning, and its walk follows the automaton of the keys as given.  encoding and
        errors: UTF-8 haystacks, as for find_all_batch (always at 4 bytes per letter)."""
        return self.find_all_batch(haystacks, algo="long", sort=sort, device=device, whole_words=whole_words,
                                   ascii_case_insensitive=ascii_case_insensitive, case_insensitive=case_insensitive,
                                   encoding=encoding, errors=errors)

    @_locked
    def find_leftmost_longest_batch(self, haystacks, *, algo: str = "auto", device: Optional[int] = None,
                                    whole_words=False, ascii_case_insensitive: bool = False,
                                    case_insensitive: bool = False, encoding: Optional[str] = None,
                                    errors: str = "strict") -> "Matches":
        """Leftmost-longest non-overlapping matches of a whole batch, selected on the GPU (input forms and result type
        of find_all_batch).  Per haystack, from the matches ``iter()`` reports: p = 0; while some match starts at or
        after p, take the smallest such start, the longest match there, and continue after its end.  Records come in
        haystack order, then end_index ascending.  This is the leftmost-longest rule of keyword extractors, not
        iter_long's: iter_long restarts from the root after every match and misses keys its walk does not pass.
        algo ("auto", "filter", "dfa") only picks the scan that finds every match; the result does not depend on it.

        whole_words (see find_all_batch): the same rule over the whole-word matches only, so a longer match inside a
        word does not hide a shorter whole word: keys ``new`` and ``new york`` on ``new yorker`` give ``new``.  A CUDA
        tensor batch then waits once more, for the number of whole-word matches.

        ascii_case_insensitive and case_insensitive (see find_all_batch): the same rule over the folded text.  Of the keys
        that fold to the same text, only the one added first is reported.

        encoding and errors (see find_all_batch): UTF-8 haystacks, decoded on the GPU; the result is that of the same
        call on the decoded list of str."""
        self._require_automaton()
        if algo not in ("auto", "filter", "dfa"):
            raise ValueError(f"algo {algo!r}: leftmost-longest takes 'auto', 'filter' or 'dfa'")
        words = self._words(whole_words)
        fold = self._fold_arg(ascii_case_insensitive, case_insensitive=case_insensitive)
        u8 = self._utf8_arg(encoding, errors)
        if u8 is not None:
            return Matches(self._leftmost_utf8(self._utf8_batch(haystacks, u8, device), algo, words, N.SELECT_LONGEST, fold),
                           self._result_values())
        b = self._batch_input(haystacks)
        if b.empty:
            rec = np.empty(0, dtype=N.MATCH_DTYPE)
        elif b.kind == "device":
            rec = self._leftmost_device(b, algo, words, fold=fold)
        elif words is not None and fold:
            rec = self._words_host(b.data, b.offsets, b.n, b.stride, algo, False, device, b.narrow, words, True, fold=fold)
        elif words is not None:
            rec = self._words_host(b.data, b.offsets, b.n, b.stride, algo, False, device, b.narrow, words, True)
        elif fold:
            rec = self._leftmost_host(b.data, b.offsets, b.n, b.stride, algo, device, b.narrow, fold=fold)
        else:
            rec = self._leftmost_host(b.data, b.offsets, b.n, b.stride, algo, device, b.narrow)
        return Matches(rec, self._result_values())

    @_locked
    def find_leftmost_first_batch(self, haystacks, *, algo: str = "auto", device: Optional[int] = None,
                                  whole_words=False, ascii_case_insensitive: bool = False,
                                  case_insensitive: bool = False, encoding: Optional[str] = None,
                                  errors: str = "strict") -> "Matches":
        """Leftmost-first non-overlapping matches of a whole batch, selected on the GPU (input forms and result type of
        find_all_batch).  Per haystack, from the matches ``iter()`` reports: p = 0; while some match starts at or after
        p, take the smallest such start, the match there whose key was added first, and continue after its end.  This is
        the rule of regex alternation (``sam|samwise`` finds ``sam`` in ``samwise``): keys earlier in the dictionary win
        at a start, but a match further left always wins.  Priority is the order in which add_word first added each key:
        add_word of a key already present keeps its place, removing a key and adding it again moves it to the end.  An
        automaton read back from pickle or save numbers its keys afresh, so its priority can differ.  Records come in
        haystack order, then end_index ascending; algo, whole_words, ascii_case_insensitive and case_insensitive as for
        find_leftmost_longest_batch (the key added first wins among keys of one folded text, as at any start).  encoding
        and errors (see find_all_batch): UTF-8 haystacks, with the result of the same call on the decoded list of str."""
        self._require_automaton()
        if algo not in ("auto", "filter", "dfa"):
            raise ValueError(f"algo {algo!r}: leftmost-first takes 'auto', 'filter' or 'dfa'")
        words = self._words(whole_words)
        fold = self._fold_arg(ascii_case_insensitive, case_insensitive=case_insensitive)
        u8 = self._utf8_arg(encoding, errors)
        if u8 is not None:
            return Matches(self._leftmost_utf8(self._utf8_batch(haystacks, u8, device), algo, words, N.SELECT_FIRST, fold),
                           self._result_values())
        b = self._batch_input(haystacks)
        if b.empty:
            rec = np.empty(0, dtype=N.MATCH_DTYPE)
        elif b.kind == "device":
            rec = self._leftmost_device(b, algo, words, N.SELECT_FIRST, fold)
        elif words is not None and fold:
            rec = self._words_host(b.data, b.offsets, b.n, b.stride, algo, False, device, b.narrow, words, True, select=N.SELECT_FIRST,
                                   fold=fold)
        elif words is not None:
            rec = self._words_host(b.data, b.offsets, b.n, b.stride, algo, False, device, b.narrow, words, True, select=N.SELECT_FIRST)
        elif fold:
            rec = self._leftmost_host(b.data, b.offsets, b.n, b.stride, algo, device, b.narrow, select=N.SELECT_FIRST, fold=fold)
        else:
            rec = self._leftmost_host(b.data, b.offsets, b.n, b.stride, algo, device, b.narrow, select=N.SELECT_FIRST)
        return Matches(rec, self._result_values())

    @_locked
    def _leftmost_host(self, flat: np.ndarray, offsets: Optional[np.ndarray], n_hay: int, stride_bytes: int, algo: str,
                       device: Optional[int], narrow: bool, select: int = N.SELECT_LONGEST, fold: int = _FOLD_NONE) -> np.ndarray:
        """acb_scan_host_leftmost (acb_scan_host_leftmost_kind for leftmost-first): upload, scan, select, copy back
        (_host_records).  fold: on the folded table, whose representatives are the winners; no alias expansion."""
        lib = self._lib
        args = (N.ptr(flat), int(flat.size), N.ptr(offsets) if offsets is not None else None, n_hay, stride_bytes)

        def scan(tb, cap, found_ref):
            if select != N.SELECT_LONGEST:
                return lib.acb_scan_host_leftmost_kind(tb, select, *args, None, -1, None, cap, found_ref, N.ALGOS[algo])
            return lib.acb_scan_host_leftmost(tb, *args, None, cap, found_ref, N.ALGOS[algo])
        return self._host_records(device, narrow, n_hay, scan, fold)

    @_locked
    def _leftmost_device(self, batch, algo: str, words: Optional[tuple] = None, select: int = N.SELECT_LONGEST,
                         fold: int = _FOLD_NONE) -> np.ndarray:
        """A CUDA tensor batch: the full scan into a device buffer, then the selection, both on torch's current stream;
        only the chosen records come back.  fold: on the folded table."""
        t = _aligned(batch.data)
        dev = _device_of(t)
        tb = self._table_for(dev, False, fold)
        with _on_device(dev) as stream:
            out, cnt, _ = self._leftmost_chosen(tb, t, batch.n, batch.stride, algo, stream, words, select)
            found = int(cnt.item())
            return out[:found].cpu().numpy().view(N.MATCH_DTYPE).reshape(-1)

    def _leftmost_chosen(self, tb, t, n: int, stride: int, algo: str, stream, words: Optional[tuple] = None,
                         select: int = N.SELECT_LONGEST, offs=None, max_letters: Optional[int] = None, narrow: bool = False):
        """The chosen records of an aligned device batch, left on the device: (records [cap, 3] int32 CUDA tensor,
        their count as an int64 CUDA tensor, cap).  Synchronises once, to size the full list; with words, the
        selection runs on the whole-word matches and a second wait sizes them (_device_matches).  select: the rule,
        acb_leftmost_longest_device or acb_leftmost_first_device.  offs, narrow: as for _device_matches, with
        max_letters the longest haystack."""
        import torch
        if max_letters is None:
            max_letters = stride // self._L
        full, m = self._device_matches(tb, t, n, stride, algo, stream, words, offs=offs, narrow=narrow)
        cap = max(m, 1)
        out = torch.empty((cap, 3), dtype=torch.int32, device=t.device)
        cnt = torch.zeros(1, dtype=torch.int64, device=t.device)
        fn = self._lib.acb_leftmost_longest_device if select == N.SELECT_LONGEST else self._lib.acb_leftmost_first_device
        N.check(fn(tb, full.data_ptr(), m, n, max_letters, out.data_ptr(), cap, cnt.data_ptr(), stream))
        return out, cnt, cap

    # ------------------------------------------------------------------ UTF-8 batches (DESIGN section 4.20)
    def _utf8_arg(self, encoding, errors) -> Optional[int]:
        """The encoding and errors arguments of the batch methods: None for haystacks of letters, else the errors kind
        of a UTF-8 batch (N.UTF8_STRICT or N.UTF8_REPLACE), checked against the automaton"""
        if errors not in ("strict", "replace"):
            raise ValueError(f"errors {errors!r}: a UTF-8 batch takes 'strict' or 'replace'")
        if encoding is None:
            if errors != "strict":
                raise ValueError("errors applies to UTF-8 haystacks: pass encoding='utf-8'")
            return None
        try:
            name = codecs.lookup(encoding).name
        except (LookupError, TypeError):
            name = None
        if name != "utf-8":
            raise ValueError(f"encoding {encoding!r}: haystacks are decoded from UTF-8 only")
        if not self._UNICODE:
            raise ValueError("encoding is for the unicode flavour: the bytes flavour matches bytes as they are, and its keys "
                             "can be UTF-8 bytes already")
        if self._key_type == KEY_SEQUENCE:
            raise ValueError("encoding needs text: KEY_SEQUENCE letters are integers, not letters")
        return N.UTF8_STRICT if errors == "strict" else N.UTF8_REPLACE

    @staticmethod
    def _utf8_upload(haystacks, device: Optional[int]):
        """The input forms of a UTF-8 batch on the GPU: (flat uint8 CUDA tensor, int64 CUDA byte offsets or None for rows
        of `stride` bytes, n, stride, the host batch as (flat, offsets or None) or None for a CUDA tensor).  A host batch
        is uploaded once, to `device`."""
        import torch
        if type(haystacks).__module__.startswith("torch") and getattr(haystacks, "is_cuda", False):
            t = haystacks
            if t.dtype != torch.uint8 or t.dim() != 2 or not t.is_contiguous():
                raise TypeError("device batches must be 2-D contiguous uint8 tensors [n_haystacks, stride_bytes]")
            return _aligned(t).reshape(-1), None, int(t.shape[0]), int(t.shape[1]), None
        if isinstance(haystacks, np.ndarray):
            if haystacks.dtype != np.uint8 or haystacks.ndim != 2 or not haystacks.flags.c_contiguous:
                raise TypeError("array batches must be 2-D C-contiguous uint8 [n_haystacks, stride_bytes]")
            (n, stride), flat, offs = haystacks.shape, haystacks.reshape(-1), None
        elif _is_pair(haystacks):
            flat = np.ascontiguousarray(haystacks[0], dtype=np.uint8).reshape(-1)
            offs = np.ascontiguousarray(haystacks[1], dtype=np.int64)
            if offs.ndim != 1 or len(offs) < 1 or offs[0] != 0 or offs[-1] != flat.size or np.any(np.diff(offs) < 0):
                raise ValueError("offsets must be non-decreasing, start at 0 and end at len(flat)")
            n, stride = len(offs) - 1, 0
        elif isinstance(haystacks, (list, tuple)):
            types = set(map(type, haystacks))
            if not types <= {bytes, bytearray}:
                if str in types:
                    raise TypeError("a UTF-8 batch holds bytes, and a str is already decoded: pass it without encoding")
                raise TypeError("a UTF-8 batch is a list or tuple of bytes or bytearray, a uint8 array [n, stride], a "
                                "(flat, offsets) pair or a uint8 CUDA tensor [n, stride]")
            n, stride = len(haystacks), 0
            offs = np.zeros(n + 1, dtype=np.int64)
            np.cumsum(np.fromiter(map(len, haystacks), dtype=np.int64, count=n), out=offs[1:])
            flat = np.frombuffer(bytearray().join(haystacks), dtype=np.uint8)
        else:
            raise TypeError("a UTF-8 batch is a list or tuple of bytes or bytearray, a uint8 array [n, stride], a "
                            "(flat, offsets) pair or a uint8 CUDA tensor [n, stride]")
        dev = f"cuda:{_default_device() if device is None else device}"
        with warnings.catch_warnings():                      # a read-only array is only read: the upload copies it
            warnings.simplefilter("ignore", UserWarning)
            t = torch.from_numpy(flat).to(dev)
            d_offs = None if offs is None else torch.from_numpy(offs).to(dev)
        return t, d_offs, n, stride, (flat, offs)

    def _utf8_batch(self, haystacks, errors: int, device: Optional[int], narrow_ok: bool = True) -> "_Utf8Batch":
        """A UTF-8 batch decoded on the GPU (acb_utf8_decode_device, acb_utf8_write_device) on torch's current stream of
        its device: at 1 byte per letter when narrow_ok and every letter is below 256, else at 4.  Waits once, for the
        info block; under "strict" an invalid sequence raises UnicodeDecodeError before pass 2."""
        import torch
        t, offs, n, stride, host = self._utf8_upload(haystacks, device)
        lib, dev, total = self._lib, _device_of(t), int(t.numel())
        need = ctypes.c_int64(0)
        N.check(lib.acb_utf8_work_bytes(total, n, ctypes.byref(need)))
        with _on_device(dev) as stream:
            work = torch.empty(int(need.value), dtype=torch.uint8, device=t.device)
            info = torch.empty(5, dtype=torch.int64, device=t.device)
            batch = (t.data_ptr() if total else None, total, None if offs is None else offs.data_ptr(), n, stride)
            N.check(lib.acb_utf8_decode_device(dev, *batch, errors, work.data_ptr(), work.numel(), info.data_ptr(), stream))
            letters, top, longest, err_start, err_end = info.tolist()
            if err_start >= 0:
                raise _utf8_error(t, host, stride, err_start, err_end)
            narrow = narrow_ok and top < 256
            width = 1 if narrow else 4
            out = torch.empty(max(letters * width, 16), dtype=torch.uint8, device=t.device)
            out_offs = torch.empty(n + 1, dtype=torch.int64, device=t.device)
            N.check(lib.acb_utf8_write_device(dev, *batch, work.data_ptr(), work.numel(), width, out.data_ptr(),
                                              out_offs.data_ptr(), stream))
        return _Utf8Batch(out[:letters * width], out_offs, n, longest, narrow)

    @_locked
    def _scan_utf8(self, b: "_Utf8Batch", algo: str, sort: bool, words: Optional[tuple], white_space: bool,
                   fold: int) -> np.ndarray:
        """find_all over a decoded UTF-8 batch: scan (skipping white space), word filter, alias expansion and sort on the
        device, as _scan_device_tensor does for a batch of rows"""
        t = b.data
        dev = _device_of(t)
        tb = self._table_for(dev, b.narrow, fold)
        if tb is None or b.n == 0 or t.numel() == 0:
            return np.empty(0, dtype=N.MATCH_DTYPE)
        skip = self._skip_set(b.narrow) if white_space else None
        with _on_device(dev) as stream:
            out, found = self._device_matches(tb, t, b.n, 0, algo, stream, words, skip, b.offsets, b.narrow)
            if fold and found and self._has_aliases(b.narrow, fold):
                out, found = self._expand_device(tb, t, b.n, out, found, stream)
            return self._device_records(tb, out, found, b.n, b.max_letters, stream, sort)

    @_locked
    def _leftmost_utf8(self, b: "_Utf8Batch", algo: str, words: Optional[tuple], select: int, fold: int) -> np.ndarray:
        """a leftmost selection over a decoded UTF-8 batch, as _leftmost_device"""
        t = b.data
        dev = _device_of(t)
        tb = self._table_for(dev, b.narrow, fold)
        if tb is None or b.n == 0 or t.numel() == 0:
            return np.empty(0, dtype=N.MATCH_DTYPE)
        with _on_device(dev) as stream:
            out, cnt, _ = self._leftmost_chosen(tb, t, b.n, 0, algo, stream, words, select, b.offsets, b.max_letters, b.narrow)
            found = int(cnt.item())
            return out[:found].cpu().numpy().view(N.MATCH_DTYPE).reshape(-1)

    @_locked
    def replacer(self, replacements=None, *, device: Optional[int] = None, leftmost_first: bool = False) -> "Replacer":
        """A `Replacer` that rewrites whole batches with the leftmost-longest matches replaced (Replacer.replace_batch);
        leftmost_first=True: the matches find_leftmost_first_batch chooses.
        replacements=None: every key is replaced by its value (STORE_ANY only); else a mapping from every key to its
        replacement, of the haystack type (bytes, str, or a tuple for KEY_SEQUENCE).  The replacements are taken when the
        replacer is made: giving a key a new value (add_word of a key already present) does not change it or make it
        stale, while adding or removing keys, or make_automaton, does."""
        self._require_automaton()
        return Replacer(self, replacements, _default_device() if device is None else device,
                        N.SELECT_FIRST if leftmost_first else N.SELECT_LONGEST)

    def dump(self):
        """(nodes, edges, fail) in the spirit of src/Automaton.c:1100-1180, with int state ids."""
        f = self.flat()
        S = f["n_states"]
        inv = {int(c): b for b, c in enumerate(f["byte_class"].tolist()) if c != 0 or f["n_classes"] == 256}
        nodes = [(s, int(f["key_of"][s] >= 0)) for s in range(S)]
        edges = []
        for c in range(f["n_classes"]):
            col = f["goto_cm"][c]
            for s in np.nonzero(col >= 0)[0].tolist():
                edges.append((s, bytes([inv[c]]), int(col[s])))
        fail = [(s, int(f["fail"][s])) for s in range(1, S)]
        return nodes, edges, fail

    # ------------------------------------------------------------------ the batch entry (new)
    @_locked
    def find_all_batch(self, haystacks, *, algo: str = "auto", sort: bool = True, device: Optional[int] = None,
                       ignore_white_space: bool = False, whole_words=False, ascii_case_insensitive: bool = False,
                       case_insensitive: bool = False, encoding: Optional[str] = None, errors: str = "strict") -> Matches:
        """Search a whole batch on the GPU.

        haystacks: a sequence of bytes / str / tuple objects (as `iter` accepts), or a 2-D
        C-contiguous uint8 array [n, stride] (bytes flavour: one haystack per row), or a pair
        (flat uint8 array, int64 byte offsets of length n+1), or a 2-D contiguous uint8 torch CUDA
        tensor [n, stride] that already lives in HBM (no host copy of the batch).

        Equivalent to ``[(h, e, v) for h, hay in enumerate(haystacks) for e, v in A.iter(hay)]``
        of the reference, returned as arrays.  ignore_white_space=True: to ``A.iter(hay, ignore_white_space=True)``
        -- letters for which libc iswspace() is true are skipped (removed on the GPU before the scan) and end_index
        still counts the letters of the original haystack.

        whole_words: keep only the whole-word matches, in the same format and order: neither the letter before the
        match nor the one after it is a word letter (a haystack edge is not one; the key's own letters do not matter,
        so ``#tag`` or ``foo bar`` work as keys).  True: re's \\w -- [0-9A-Za-z_] for the bytes flavour (flashtext's
        default; the bytes of a UTF-8 letter such as b"\\xc3\\xa9" are not word letters, so b"caf" is a whole word in
        b"caf\\xc3\\xa9": give bytes 0x80-0xFF as word letters for UTF-8 text), isalnum() or "_" for the unicode
        flavour.  bytes (bytes flavour) or str (unicode flavour): exactly these word letters; empty: none, every match
        is kept.  The matches are filtered on the GPU after the scan; a CUDA tensor batch then waits once more, for
        their number.  ValueError with ignore_white_space, algo="long" or a KEY_SEQUENCE automaton.

        ascii_case_insensitive: the 26 ASCII letters match either case and nothing else folds -- a byte 0x41-0x5A equals
        itself + 0x20 (bytes flavour), a code point 0x41-0x5A equals itself + 0x20 (unicode flavour; É and é, or Ł and
        š, stay distinct).  Every key whose folded text occurs is reported, so keys ``abc`` and ``ABC`` both match in
        ``xAbCx``; keys of one length at one end (case variants of each other) come in ascending key id.  end_index and
        the whole-word test are those of the text as given.  The text is folded on the GPU; the caller's copy is not
        changed.  ValueError with ignore_white_space, algo="long" or a KEY_SEQUENCE automaton.

        case_insensitive (unicode flavour): letters match when Unicode simple case folding maps them to the same letter
        (`_unicode_fold_map`, from the running Python's unicodedata): ``Müller`` matches ``MÜLLER``, ``Σοφία`` matches
        ``ΣΟΦΊΑ``, ``Straße`` matches ``STRAẞE``, and K, k and the Kelvin sign match each other, also in a latin-1 batch.
        One letter folds to one letter only: ``ß`` does not match ``ss`` nor ``ﬁ`` ``fi``; there is no Turkic rule (``ı``
        and ``İ`` match neither ``i`` nor ``I``) and no normalisation (``é`` does not match ``e`` + U+0301).  Everything
        else is as for ascii_case_insensitive: every key whose folded text occurs, case variants in ascending key id,
        end_index and whole words of the text as given, the text folded on the GPU and the caller's copy unchanged.
        ValueError for the bytes flavour (bytes have no known encoding: use ascii_case_insensitive), together with
        ascii_case_insensitive, with ignore_white_space, algo="long" or a KEY_SEQUENCE automaton.

        encoding="utf-8" (unicode flavour, KEY_STRING keys; any name codecs.lookup gives as utf-8): the haystacks are
        UTF-8 bytes -- a list or tuple of bytes or bytearray (a str item raises TypeError), a (flat uint8, int64 byte
        offsets) pair, a C-contiguous uint8 array [n, stride] of one haystack per row (NUL bytes included) or a
        contiguous uint8 CUDA tensor [n, stride] -- decoded on the GPU.  The result is exactly that of the same call on
        ``[h.decode("utf-8", errors) for h in haystacks]``: end_index counts letters (code points).  errors="strict"
        raises the UnicodeDecodeError CPython raises for the first haystack with an invalid sequence (its bytes, start
        and end) before anything is scanned; errors="replace" decodes each invalid sequence to one U+FFFD, as CPython
        does, so a key holding U+FFFD matches it.  A batch whose letters are all below 256 runs on the latin-1 automaton
        at 1 byte per letter (not with algo="long"); the width changes speed, never results.  Host input is uploaded
        once and searched unpipelined.  ValueError for the bytes flavour (it matches the bytes themselves), KEY_SEQUENCE
        automata, another encoding, or errors other than "strict" and "replace"; errors other than "strict" also needs
        an encoding.
        """
        self._require_automaton()
        if ignore_white_space and algo == "long":
            raise ValueError("iter_long has no ignore_white_space option")
        words = self._words(whole_words)
        if words is not None and ignore_white_space:
            raise ValueError("whole_words cannot be combined with ignore_white_space")
        if words is not None and algo == "long":
            raise ValueError("whole_words cannot be combined with algo='long': iter_long's walk picks its matches itself")
        fold = self._fold_arg(ascii_case_insensitive, algo, ignore_white_space, case_insensitive)
        u8 = self._utf8_arg(encoding, errors)
        if u8 is not None:
            b = self._utf8_batch(haystacks, u8, device, narrow_ok=algo != "long")
            return Matches(self._scan_utf8(b, algo, sort, words, ignore_white_space, fold), self._result_values())
        b = self._batch_input(haystacks, narrow_ok=algo != "long")
        if b.empty:
            rec = np.empty(0, dtype=N.MATCH_DTYPE)
        elif b.kind == "device":
            rec = self._scan_device_tensor(b, algo, sort, words, ignore_white_space, fold)
        elif words is not None and fold:
            rec = self._words_host(b.data, b.offsets, b.n, b.stride, algo, sort, device, b.narrow, words, False, fold=fold)
        elif words is not None:
            rec = self._words_host(b.data, b.offsets, b.n, b.stride, algo, sort, device, b.narrow, words, False)
        elif ignore_white_space:
            rec = self._scan_skip(b, algo, sort, device)
        elif fold:
            rec = self._scan_flat(b.data, b.offsets, b.n, b.stride, algo=algo, sort=sort, device=device, narrow=b.narrow, fold=fold)
        else:
            rec = self._scan_flat(b.data, b.offsets, b.n, b.stride, algo=algo, sort=sort, device=device, narrow=b.narrow)
        return Matches(rec, self._result_values())

    def _batch_input(self, haystacks, narrow_ok: bool = True, required: bool = True) -> "_Batch":
        """The input forms of find_all_batch, checked and laid out for a scan (_Batch).  narrow: the buffer holds the
        1-byte letters of the latin-1 automaton (unicode flavour, only where narrow_ok).  required=False: an item of the
        wrong type raises the TypeError of the dict-like methods instead of iter()'s."""
        L = self._L
        if type(haystacks).__module__.startswith("torch") and getattr(haystacks, "is_cuda", False):
            return _Batch("device", haystacks, None, *self._device_batch_shape(haystacks), False)
        if isinstance(haystacks, np.ndarray):
            if haystacks.dtype != np.uint8 or haystacks.ndim != 2 or not haystacks.flags.c_contiguous:
                raise TypeError("array batches must be 2-D C-contiguous uint8 [n_haystacks, stride_bytes]")
            n, stride = haystacks.shape
            if stride % L:
                raise ValueError("row length must be a multiple of the letter width")
            return _Batch("host", haystacks.reshape(-1), None, n, stride, False)
        if _is_pair(haystacks):
            flat = np.ascontiguousarray(haystacks[0], dtype=np.uint8).reshape(-1)
            offs = np.ascontiguousarray(haystacks[1], dtype=np.int64)
            if offs.ndim != 1 or len(offs) < 1 or offs[0] != 0 or offs[-1] != flat.size or np.any(np.diff(offs) < 0) or np.any(offs % L):
                raise ValueError("offsets must be non-decreasing multiples of the letter width, start at 0 and end at len(flat)")
            return _Batch("host", flat, offs, len(offs) - 1, 0, False)
        # the latin-1 automaton finds exactly the matches of a latin-1 haystack -- all of them.  iter_long's walk is
        # different: which match it keeps depends on the whole trie (a non-latin-1 key whose prefix is latin-1 adds
        # nodes the walk passes through, src/AutomatonSearchIterLong.c:118-126), so it always runs on the full one
        # the common drop-in inputs, a list of bytes objects or (4-byte letters only) of str objects: one join instead
        # of an array per haystack.  utf-32 encodes every code point by itself, so the joined buffer holds exactly the
        # bytes of the items encoded one by one
        wide_str = self._UNICODE and not narrow_ok
        if self._key_type == KEY_STRING and (wide_str or not self._UNICODE) and isinstance(haystacks, (list, tuple)) \
                and haystacks and set(map(type, haystacks)) == {str if wide_str else bytes}:   # C-level pass, 3 x faster than all()
            n = len(haystacks)
            offs = np.zeros(n + 1, dtype=np.int64)
            np.cumsum(np.fromiter(map(len, haystacks), dtype=np.int64, count=n), out=offs[1:])
            if wide_str:
                offs *= 4
                flat = "".join(haystacks).encode("utf-32-le", "surrogatepass")
            else:
                flat = b"".join(haystacks)
            return _Batch("host", np.frombuffer(flat, dtype=np.uint8), offs, n, 0, False)
        get = self._hay_letters if narrow_ok else self._letters
        letters = [get(h, required=required) for h in haystacks]
        narrow = self._uses_narrow() and len(letters) > 0 and all(a.dtype == np.uint8 for a in letters)
        if self._uses_narrow() and not narrow:                   # mixed batch: everything at 4 bytes per letter
            letters = [a.astype("<u4") if a.dtype == np.uint8 else a for a in letters]
        parts = [np.ascontiguousarray(a).view(np.uint8) for a in letters]
        n = len(parts)
        lens = np.fromiter((p.size for p in parts), dtype=np.int64, count=n)
        offs = np.zeros(n + 1, dtype=np.int64)
        np.cumsum(lens, out=offs[1:])
        flat = np.concatenate(parts) if n else np.empty(0, dtype=np.uint8)
        return _Batch("host", flat, offs, n, 0, narrow)

    def stream_batch(self, n_streams: int, *, long: bool = False, algo: str = "auto",
                     device: Optional[int] = None, ignore_white_space: bool = False,
                     leftmost_longest: bool = False, whole_words=False, leftmost_first: bool = False,
                     encoding: Optional[str] = None, errors: str = "strict") -> "StreamBatch":
        """`n_streams` independent streams searched chunk by chunk, the next chunk of many of them in one GPU call
        (StreamBatch.feed).  long=False: stream s reports what the reference's ``iter(c0)`` ... ``.set(c1)`` ...
        reports over its chunks -- every match, also those across chunk boundaries; long=True: what
        ``iter_long(c0)`` ... ``.set(c1)`` reports.  What a stream carries from one chunk to the next stays in HBM.
        ignore_white_space=True (find_all batches only): what ``iter(c0, ignore_white_space=True)`` ... ``.set(c1)``
        ... reports; positions still count every letter, and a key that white space splits across chunks is found.
        leftmost_longest=True: what `find_leftmost_longest_batch` reports for each stream's whole text, delivered as
        soon as no later letter can change it (see StreamBatch.finish); leftmost_first=True: the same for
        `find_leftmost_first_batch` (not with leftmost_longest, long or ignore_white_space).
        whole_words (see find_all_batch; not with long=True or ignore_white_space=True): only whole-word matches, what
        find_all_batch or find_leftmost_longest_batch reports with the same option for each stream's whole text.  A
        match is reported once the letter after it has arrived (or by `finish`), so a stream holds back one letter more.

        Unicode flavour: streams are always scanned at 4 bytes per letter (a stream can switch between latin-1 and
        wider chunks, so the latin-1 automaton is not used).

        encoding="utf-8" (unicode flavour, KEY_STRING keys; errors "strict" or "replace"): the chunks are UTF-8 bytes,
        decoded on the GPU, in the input forms of find_all_batch's UTF-8 batches.  A letter may be split across chunks:
        each stream holds back the bytes of a letter it has not finished (``pending``, at most 3) until its next feed or
        `finish`.  The batch reports exactly what the same batch of `str` reports when each chunk is replaced by
        ``dec.decode(chunk)`` of an incremental decoder per stream (``codecs.getincrementaldecoder("utf-8")(errors)``)
        and `finish` is preceded by ``dec.decode(b"", final=True)``; end_index and positions count letters.  So over all
        feeds and `finish` a stream gets what the whole-batch method with encoding="utf-8" gives for the concatenation
        of its chunks.  Such a find_all batch (also long=True and ignore_white_space=True) has a `finish` too."""
        return self._stream_batch(n_streams, long, algo, device, ignore_white_space, leftmost_longest, whole_words,
                                  leftmost_first, _FOLD_NONE, encoding, errors)

    def ascii_case_insensitive_stream_batch(self, n_streams: int, *, algo: str = "auto", device: Optional[int] = None,
                                            leftmost_longest: bool = False, leftmost_first: bool = False,
                                            whole_words=False, encoding: Optional[str] = None,
                                            errors: str = "strict") -> "StreamBatch":
        """`stream_batch` with ASCII case-insensitive matching: over all feeds (and `finish`) of a stream, what
        find_all_batch, find_leftmost_longest_batch or find_leftmost_first_batch reports for its whole text with
        ascii_case_insensitive=True and the same whole_words.  A find_all batch reports every key whose folded text
        occurs, keys of one length at one end in ascending id; a leftmost batch reports, of the keys that fold to one
        text, the one added first.  Matches are released at the same points as by the stream_batch of the same options,
        and the word test reads the letters as given.  Takes neither long nor ignore_white_space; not for KEY_SEQUENCE
        automata.  The returned StreamBatch has ``ascii_case_insensitive`` True.  encoding and errors: UTF-8 chunks, as
        for stream_batch."""
        return self._stream_batch(n_streams, False, algo, device, False, leftmost_longest, whole_words, leftmost_first,
                                  _FOLD_ASCII, encoding, errors)

    def case_insensitive_stream_batch(self, n_streams: int, *, algo: str = "auto", device: Optional[int] = None,
                                      leftmost_longest: bool = False, leftmost_first: bool = False,
                                      whole_words=False, encoding: Optional[str] = None,
                                      errors: str = "strict") -> "StreamBatch":
        """`stream_batch` with Unicode case-insensitive matching (unicode flavour): over all feeds (and `finish`) of a
        stream, what find_all_batch, find_leftmost_longest_batch or find_leftmost_first_batch reports for its whole text
        with case_insensitive=True and the same whole_words.  A find_all batch reports every key whose folded text occurs,
        keys of one length at one end in ascending id; a leftmost batch reports, of the keys that fold to one text, the
        one added first.  Matches are released at the same points as by the stream_batch of the same options, and the
        word test reads the letters as given.  Takes neither long nor ignore_white_space; not for the bytes flavour or
        KEY_SEQUENCE automata.  The returned StreamBatch has ``case_insensitive`` True.  encoding and errors: UTF-8
        chunks, as for stream_batch."""
        return self._stream_batch(n_streams, False, algo, device, False, leftmost_longest, whole_words, leftmost_first,
                                  _FOLD_UNICODE, encoding, errors)

    @_locked
    def _stream_batch(self, n_streams: int, long: bool, algo: str, device: Optional[int], ignore_white_space: bool,
                      leftmost_longest: bool, whole_words, leftmost_first: bool, fold: int, encoding: Optional[str] = None,
                      errors: str = "strict") -> "StreamBatch":
        """The argument check and constructor of stream_batch, ascii_case_insensitive_stream_batch and
        case_insensitive_stream_batch (fold: the fold kind)"""
        self._require_automaton()
        u8 = self._utf8_arg(encoding, errors)
        self._fold_arg(fold == _FOLD_ASCII, case_insensitive=fold == _FOLD_UNICODE)
        n_streams = operator.index(n_streams)
        if n_streams < 0:
            raise ValueError("n_streams must not be negative")
        words = self._words(whole_words)
        if words is not None and (long or ignore_white_space):
            raise ValueError("whole_words stream batches take neither long=True nor ignore_white_space=True")
        if leftmost_longest and (long or ignore_white_space):
            raise ValueError("leftmost_longest stream batches take neither long=True nor ignore_white_space=True")
        if leftmost_first and (leftmost_longest or long or ignore_white_space):
            raise ValueError("leftmost_first stream batches take none of leftmost_longest, long=True and ignore_white_space=True")
        if algo not in (("auto", "long") if long else ("auto", "filter", "dfa")):
            raise ValueError(f"algo {algo!r} does not fit a {'long' if long else 'find_all'} stream batch")
        if long and ignore_white_space:
            raise ValueError("iter_long has no ignore_white_space option")
        skip = self._skip_set(False) if ignore_white_space else None
        return StreamBatch(self, n_streams, bool(long), algo, _default_device() if device is None else device, skip,
                           bool(leftmost_longest), words, bool(leftmost_first), fold, u8, errors)

    # ------------------------------------------------------------------ batch lookups (new)
    # exists / match / longest_prefix / get for a whole batch of keys, in one GPU call (acb_lookup_*).  `keys` takes the
    # input forms of find_all_batch.  The walk always runs on the full table: a latin-1 key can be a prefix of a key
    # that is not latin-1, and the latin-1 automaton lacks those nodes.
    def exists_batch(self, keys, *, device: Optional[int] = None):
        """``[A.exists(k) for k in keys]`` as bool[n] (a bool CUDA tensor, not synchronised, for a CUDA tensor batch)."""
        key_id, _, _ = self._lookup_batch(keys, device)
        return key_id >= 0

    def match_batch(self, keys, *, device: Optional[int] = None):
        """``[A.match(k) for k in keys]`` as bool[n] (a bool CUDA tensor, not synchronised, for a CUDA tensor batch)."""
        _, prefix, lens = self._lookup_batch(keys, device)
        return prefix == lens

    def longest_prefix_batch(self, keys, *, device: Optional[int] = None):
        """``[A.longest_prefix(k) for k in keys]`` as int64[n] (an int64 CUDA tensor, not synchronised, for a CUDA
        tensor batch)."""
        _, prefix, _ = self._lookup_batch(keys, device)
        return prefix.astype(np.int64) if isinstance(prefix, np.ndarray) else prefix.long()

    def get_batch(self, keys, default=_MISSING, *, device: Optional[int] = None) -> list:
        """``[A.get(k[, default]) for k in keys]``: a list of values, read when the call returns.  Without a default,
        KeyError of the first key that is missing."""
        if not isinstance(keys, (list, tuple, np.ndarray)) and not type(keys).__module__.startswith("torch"):
            keys = list(keys)                                   # an iterator: kept, for the KeyError
        with self._gpu_lock:                                    # the ids and the values of one key set
            key_id, _, _ = self._lookup_batch(keys, device)
            if not isinstance(key_id, np.ndarray):
                key_id = key_id.cpu().numpy()                  # synchronises torch's current stream
            values = self._values
            if default is Automaton._MISSING:
                miss = np.flatnonzero(key_id < 0)
                if miss.size:
                    raise KeyError(self._batch_key(keys, int(miss[0])))
            else:
                values = values + [default]                     # key_id -1 picks it
            return list(map(values.__getitem__, key_id.tolist()))

    @_locked
    def _lookup_batch(self, keys, device: Optional[int]):
        """(key_id int32[n], prefix int32[n], length of every key in letters) of a batch of keys: numpy arrays, or for
        a CUDA tensor int32 CUDA tensors computed on torch's current stream and one length for all rows."""
        self._require_automaton()
        kind, data, offs, n, stride, _ = self._batch_input(keys, narrow_ok=False, required=False)
        if kind == "device":
            import torch
            t = data
            key_id = torch.empty(n, dtype=torch.int32, device=t.device)
            prefix = torch.empty(n, dtype=torch.int32, device=t.device)
            if n:
                dev = _device_of(t)
                tb = self._ensure_table(dev)
                with _on_device(dev) as stream:
                    N.check(self._lib.acb_lookup_device(tb, t.data_ptr() if stride else None, n * stride, None, n, stride,
                                                        key_id.data_ptr(), prefix.data_ptr(), stream))
            return key_id, prefix, stride // self._L
        key_id, prefix = self._lookup_host(data, offs, n, stride, device)
        lens = (np.diff(offs) if offs is not None else np.full(n, stride, dtype=np.int64)) // self._L
        return key_id, prefix, lens

    def _lookup_host(self, flat: np.ndarray, offsets: Optional[np.ndarray], n: int, stride_bytes: int,
                     device: Optional[int]):
        """acb_lookup_host over a host batch -> (key_id int32[n], prefix int32[n])"""
        key_id = np.empty(n, dtype=np.int32)
        prefix = np.empty(n, dtype=np.int32)
        if n:
            tb = self._ensure_table(device)
            N.check(self._lib.acb_lookup_host(tb, N.ptr(flat) if flat.size else None, int(flat.size),
                                              N.ptr(offsets) if offsets is not None else None, n, stride_bytes,
                                              N.ptr(key_id), N.ptr(prefix)))
        return key_id, prefix

    def _batch_key(self, keys, i: int):
        """key i of a batch as the dict-like methods take it (for KeyError)"""
        if _is_pair(keys):
            flat, offs = keys
            raw = np.ascontiguousarray(flat, dtype=np.uint8).reshape(-1)[int(offs[i]):int(offs[i + 1])].tobytes()
        elif isinstance(keys, (list, tuple)):
            return keys[i]
        elif isinstance(keys, np.ndarray):
            raw = keys[i].tobytes()
        else:
            raw = keys[i].cpu().numpy().tobytes()
        if self._key_type == KEY_SEQUENCE:
            return tuple(np.frombuffer(raw, dtype=_LETTER_DTYPE[self._L]).tolist())
        if self._UNICODE:
            try:
                return raw.decode("utf-32-le", "surrogatepass")
            except UnicodeDecodeError:                          # letters beyond U+10FFFF: no str holds them
                return raw
        return raw

    # ------------------------------------------------------------------ batch keys / values / items (new)
    # keys(pattern, wildcard, how) for a whole batch of patterns, in one GPU call (acb_select_*).  `patterns` takes the
    # input forms of find_all_batch; wildcard and how are those of keys() and apply to every pattern.  The walk runs on
    # the full table, as the lookups do: the latin-1 table lacks the nodes of keys that are not latin-1.
    def keys_batch(self, patterns, wildcard=None, how=MATCH_EXACT_LENGTH, *, device: Optional[int] = None) -> list:
        """``[list(A.keys(p, wildcard, how)) for p in patterns]``, read when the call returns."""
        with self._gpu_lock:                                    # the ids and the keys of one key set
            ko = self._key_objs
            return [list(map(ko.__getitem__, ids)) for ids in self._select_lists(patterns, wildcard, how, device)]

    def values_batch(self, patterns, wildcard=None, how=MATCH_EXACT_LENGTH, *, device: Optional[int] = None) -> list:
        """``[list(A.values(p, wildcard, how)) for p in patterns]``, read when the call returns."""
        with self._gpu_lock:
            vals = self._values
            return [list(map(vals.__getitem__, ids)) for ids in self._select_lists(patterns, wildcard, how, device)]

    def items_batch(self, patterns, wildcard=None, how=MATCH_EXACT_LENGTH, *, device: Optional[int] = None) -> list:
        """``[list(A.items(p, wildcard, how)) for p in patterns]``, read when the call returns."""
        with self._gpu_lock:
            ko, vals = self._key_objs, self._values
            return [[(ko[k], vals[k]) for k in ids] for ids in self._select_lists(patterns, wildcard, how, device)]

    def _select_lists(self, patterns, wildcard, how, device):
        """the key ids of every pattern, as lists"""
        offs, key_id = self.select_batch(patterns, wildcard, how, device=device)
        if not isinstance(key_id, np.ndarray):
            offs, key_id = offs.cpu().numpy(), key_id.cpu().numpy()
        ids = key_id.tolist()
        bounds = offs.tolist()
        return [ids[bounds[i]:bounds[i + 1]] for i in range(len(bounds) - 1)]

    @_locked
    def select_batch(self, patterns, wildcard=None, how=MATCH_EXACT_LENGTH, *, device: Optional[int] = None):
        """The keys of every pattern as (offsets int64[n+1], key_id int32[m]): the ids of the keys that
        ``A.keys(patterns[i], wildcard, how)`` yields are ``key_id[offsets[i]:offsets[i+1]]``, in its order.  numpy
        arrays for a host batch; for a CUDA tensor batch, CUDA tensors computed on torch's current stream.  The size of
        the output depends on the data, so the call synchronises once to learn it.  Arguments are checked as keys()
        checks them: the first pattern, then wildcard, then how, then the other patterns."""
        self._require_automaton()
        first = patterns[0] if isinstance(patterns, (list, tuple)) and patterns and not _is_pair(patterns) else None
        _, w, how = self._select_args((first, wildcard, how))
        w = -1 if w is None else w
        kind, data, offs, n, stride, _ = self._batch_input(patterns, narrow_ok=False, required=False)
        if kind == "device":
            return self._select_device(data, n, stride, w, how)
        return self._select_host(data, offs, n, stride, w, how, device)

    def _select_device(self, t, n: int, stride: int, wildcard: int, how: int):
        import torch
        out_offs = torch.empty(n + 1, dtype=torch.int64, device=t.device)
        total = torch.empty(1, dtype=torch.int64, device=t.device)
        dev = _device_of(t)
        tb = self._select_table(dev)
        with _on_device(dev) as stream:
            args = (tb, t.data_ptr() if n * stride else None, n * stride, None, n, stride, wildcard, how, out_offs.data_ptr())
            N.check(self._lib.acb_select_device(*args, None, 0, total.data_ptr(), stream))
            m = int(total.item())                               # the one synchronisation: the size of the output
            key_id = torch.empty(m, dtype=torch.int32, device=t.device)
            if m:
                N.check(self._lib.acb_select_device(*args, key_id.data_ptr(), m, total.data_ptr(), stream))
        return out_offs, key_id

    def _select_host(self, flat: np.ndarray, offsets: Optional[np.ndarray], n: int, stride_bytes: int, wildcard: int,
                     how: int, device: Optional[int]):
        """acb_select_host over a host batch -> (offsets int64[n+1], key_id int32[m])"""
        out_offs = np.zeros(n + 1, dtype=np.int64)
        if n == 0:
            return out_offs, np.empty(0, dtype=np.int32)
        tb = self._select_table(device)
        total = ctypes.c_int64(0)
        args = (tb, N.ptr(flat) if flat.size else None, int(flat.size), N.ptr(offsets) if offsets is not None else None,
                n, stride_bytes, wildcard, how, N.ptr(out_offs))
        rc = self._lib.acb_select_host(*args, None, 0, ctypes.byref(total))
        if rc == N.ACB_EOVERFLOW:                               # the ids are written by a second call of the right size
            key_id = np.empty(total.value, dtype=np.int32)
            rc = self._lib.acb_select_host(*args, N.ptr(key_id), total.value, ctypes.byref(total))
        else:
            key_id = np.empty(0, dtype=np.int32)
        N.check(rc)
        return out_offs, key_id

    def _select_table(self, device: Optional[int]):
        """the full table of `device`, with the key ranges of the select calls on it"""
        tb = self._ensure_table(device)
        N.check(self._lib.acb_table_upload_key_ranges(tb, self._trie))
        return tb

    @_locked
    def key_ranges(self) -> dict:
        """White-box view of the key order as ranges over the flat tables (acb_trie_key_ranges), numpy copies: order
        (key ids in keys() order), lo / cnt per state, child_ptr / child (letter-children, youngest first)."""
        fv = N.FlatView()
        N.check(self._lib.acb_trie_flat_view(self._trie, ctypes.byref(fv)))
        S = fv.n_states
        order = np.empty(max(len(self), 1), dtype=np.int32)
        lo, cnt, child = (np.empty(S, dtype=np.int32) for _ in range(3))
        child_ptr = np.empty(S + 1, dtype=np.int32)
        e = ctypes.c_int64(0)
        N.check(self._lib.acb_trie_key_ranges(self._trie, N.ptr(order), N.ptr(lo), N.ptr(cnt), N.ptr(child_ptr),
                                              N.ptr(child), ctypes.byref(e)))
        return dict(order=order[:len(self)], lo=lo, cnt=cnt, child_ptr=child_ptr, child=child[:e.value])


class _Streams:
    """What StreamBatch and ReplaceStream share: the native stream batch `_ss`, reached only through `_native`, the
    check that the key set has not changed, stream ids, `reset` and `positions`; for UTF-8 batches the carried bytes
    `_carry` (acb_utf8_carry), `pending` and the staging and decoding of a feed (_utf8_stage)."""

    def _init_utf8(self, u8: Optional[int], errors: str) -> None:
        """encoding, errors and the native carries of a UTF-8 batch (u8: its errors kind, None for letters)"""
        self._u8 = u8
        self.encoding = None if u8 is None else "utf-8"
        self.errors = errors
        self._carry = None
        if u8 is not None:
            c = ctypes.c_void_p()
            N.check(self._A._lib.acb_utf8_carry_new(self._device, self.n_streams, ctypes.byref(c)))
            self._carry = c

    def __del__(self):
        try:
            if getattr(self, "_ss", None) is not None:
                self._native("free")
                self._ss = None
            if getattr(self, "_carry", None) is not None:
                self._A._lib.acb_utf8_carry_free(self._carry)
                self._carry = None
        except Exception:                                   # interpreter shutdown
            pass

    def _check(self):
        if self._version != self._A._version:
            raise ValueError("underlaying automaton has changed, iterator is not valid anymore")

    def _native(self, op: str, *args):
        """The calls both kinds of native stream batch take: free;  reset(ids int32 or None);  positions ->
        int64[n_streams]"""
        lib = self._A._lib
        if op == "free":
            lib.acb_streams_free(self._ss)
            return None
        if op == "reset":
            ids, = args
            N.check(lib.acb_streams_reset(self._ss, None if ids is None else N.ptr(ids), 0 if ids is None else len(ids)))
            return None
        out = np.empty(max(self.n_streams, 1), dtype=np.int64)                  # positions
        N.check(lib.acb_streams_positions(self._ss, N.ptr(out), self.n_streams))
        return out[:self.n_streams]

    def _table(self):
        """(the table every call of this batch runs on, whether it is folded): the automaton's full table, or for a
        case-insensitive batch the folded one of its fold kind -- the full one when there is no key, which matches
        nothing either way"""
        A = self._A
        tb = A._table_for(self._device, False, self._fold) if self._fold else None
        return (A._ensure_table(self._device), False) if tb is None else (tb, True)

    def _ids(self, ids, n: int) -> Optional[np.ndarray]:
        if ids is None:
            if n > self.n_streams:
                raise ValueError(f"{n} chunks for {self.n_streams} streams: pass ids")
            return None
        a = np.asarray(ids)
        if a.ndim != 1 or len(a) != n or (a.size and not np.issubdtype(a.dtype, np.integer)):
            raise ValueError(f"ids must be {n} integers, one per chunk")
        if a.size and (a.min() < 0 or a.max() >= self.n_streams):
            raise ValueError(f"stream ids must lie in [0, {self.n_streams})")
        if len(np.unique(a)) != len(a):
            raise ValueError("a stream id is given twice")
        return np.ascontiguousarray(a, dtype=np.int32)

    def reset(self, ids=None) -> None:
        """Streams `ids` (default: all) back to their start, as ``set(x, reset=True)`` does: position 0, nothing carried
        over or held back (for a UTF-8 batch, no pending bytes either)."""
        with self._A._gpu_lock:
            self._check()
            if ids is not None:
                a = np.asarray(ids)
                if a.ndim != 1 or (a.size and not np.issubdtype(a.dtype, np.integer)) or (a.size and (a.min() < 0 or a.max() >= self.n_streams)):
                    raise ValueError(f"stream ids must be integers in [0, {self.n_streams})")
                ids = np.unique(a).astype(np.int32)
            self._reset(ids)

    def _reset(self, ids: Optional[np.ndarray]) -> None:
        """reset of streams ids (int32, distinct; None: all), under the lock"""
        self._native("reset", ids)
        if self._carry is not None:
            N.check(self._A._lib.acb_utf8_carry_reset(self._carry, None if ids is None else N.ptr(ids),
                                                      0 if ids is None else len(ids)))
        self._restart(slice(None) if ids is None else ids)

    def _restart(self, streams) -> None:
        """`streams` (an index into the streams) are back at position 0: for what the Python side keeps per stream"""

    @property
    def positions(self) -> np.ndarray:
        """int64[n_streams]: letters every stream has consumed since its start, its last reset or its last finish (a
        copy)."""
        with self._A._gpu_lock:
            return self._native("positions")

    @property
    def pending(self) -> np.ndarray:
        """int64[n_streams]: the bytes (0 to 3) each stream of a UTF-8 batch holds back because they begin a letter its
        text has not finished yet -- what its incremental decoder would keep; not counted in `positions`.  Zeros for a
        batch of letters.  A copy."""
        with self._A._gpu_lock:
            out = np.zeros(max(self.n_streams, 1), dtype=np.int64)
            if self._carry is not None:
                N.check(self._A._lib.acb_utf8_carry_pending(self._carry, N.ptr(out), len(out)))
            return out[:self.n_streams]

    def _utf8_stage(self, chunks, ids, final: bool) -> "_Utf8Feed":
        """A UTF-8 feed's chunks (the input forms of a UTF-8 batch; in a list, None is an empty chunk) behind their
        streams' carried bytes, staged (acb_utf8_carry_stage_device) and decoded to 4-byte letters on the GPU, on torch's
        current stream.  Waits once, for the decode's info block.  Under "strict" an invalid sequence raises
        UnicodeDecodeError for the first chunk that holds one, as its stream's incremental decoder raises it; nothing is
        committed until _utf8_commit."""
        import torch
        A = self._A
        lib = A._lib
        if isinstance(chunks, (list, tuple)) and not _is_pair(chunks):
            chunks = [b"" if c is None else c for c in chunks]
        t, offs, n, stride, host = A._utf8_upload(chunks, self._device)
        if host is None and _device_of(t) != self._device:
            raise ValueError(f"chunks on cuda:{_device_of(t)} for a stream batch on cuda:{self._device}")
        ids32 = self._ids(ids, n)
        total = int(t.numel())
        span = total + 3 * n                               # the most staged bytes: every chunk behind 3 carried ones
        with _on_device(self._device) as stream:
            d_ids = None if ids32 is None else torch.from_numpy(ids32).to(t.device)
            staged = torch.empty(max(span, 16), dtype=torch.uint8, device=t.device)
            soffs = torch.empty(n + 1, dtype=torch.int64, device=t.device)
            N.check(lib.acb_utf8_carry_stage_device(self._carry, t.data_ptr() if total else None, total,
                                                    None if offs is None else offs.data_ptr(), n, stride,
                                                    None if d_ids is None else d_ids.data_ptr(), int(final),
                                                    staged.data_ptr(), staged.numel(), soffs.data_ptr(), stream))
            need = ctypes.c_int64(0)
            N.check(lib.acb_utf8_work_bytes(span, n, ctypes.byref(need)))
            work = torch.empty(int(need.value), dtype=torch.uint8, device=t.device)
            info = torch.empty(6, dtype=torch.int64, device=t.device)
            batch = (staged.data_ptr(), span, soffs.data_ptr(), n, 0)
            N.check(lib.acb_utf8_decode_device(self._device, *batch, self._u8, work.data_ptr(), work.numel(), info.data_ptr(),
                                               stream))
            info[5:].copy_(soffs[n:])                      # the staged size, read with the info block
            letters, _, longest, err_start, err_end, staged_total = info.tolist()
            if err_start >= 0:
                raise self._utf8_stream_error(t, host, stride, soffs.cpu().numpy(), ids32, err_start, err_end)
            out = torch.empty(max((letters + span - staged_total) * 4, 16), dtype=torch.uint8, device=t.device)
            out_offs = torch.empty(n + 1, dtype=torch.int64, device=t.device)
            N.check(lib.acb_utf8_write_device(self._device, *batch, work.data_ptr(), work.numel(), 4, out.data_ptr(),
                                              out_offs.data_ptr(), stream))
        return _Utf8Feed(out[:letters * 4], out_offs, n, longest, ids32, d_ids)

    def _utf8_stream_error(self, t, host, stride: int, soffs: np.ndarray, ids32, start: int, end: int) -> UnicodeDecodeError:
        """The UnicodeDecodeError of the invalid sequence at staged bytes [start, end): its object is the carried bytes
        of the chunk's stream followed by the chunk, as the stream's incremental decoder raises it"""
        h = int(np.searchsorted(soffs, start, side="right")) - 1
        if host is not None and host[1] is not None:
            chunk = host[0][host[1][h]:host[1][h + 1]]
        else:
            chunk = host[0][h * stride:(h + 1) * stride] if host is not None else t[h * stride:(h + 1) * stride].cpu().numpy()
        held, k = (ctypes.c_uint8 * 3)(), ctypes.c_int32(0)
        N.check(self._A._lib.acb_utf8_carry_bytes(self._carry, h if ids32 is None else int(ids32[h]), held, ctypes.byref(k)))
        base = int(soffs[h])
        return _decode_error(bytes(held)[:k.value] + chunk.tobytes(), start - base, end - base)

    def _utf8_commit(self, f: "_Utf8Feed") -> None:
        """After a UTF-8 feed succeeded: the carries it staged become the streams' (acb_utf8_carry_commit_device)"""
        with _on_device(self._device) as stream:
            N.check(self._A._lib.acb_utf8_carry_commit_device(self._carry, None if f.d_ids is None else f.d_ids.data_ptr(), f.n,
                                                              stream))


class StreamBatch(_Streams):
    """Result of `Automaton.stream_batch()`: the carry-over of `n_streams` streams, kept on the GPU.

    ``feed(chunks, ids=None)`` hands over the next chunk of some streams and returns a `Matches` whose ``hay_id`` is
    the stream id and whose ``end_index`` (int64) is the position of the match's last letter in the whole stream,
    counted from its start or its last `reset` -- exact past 2^31, unlike the reference's C int (SURVEY A7).  Records
    come in chunk order, then end_index ascending, then longest key first.  ``positions`` is the number of letters
    every stream has consumed.  A stream batch belongs to the key set it was made for: after the key set changes,
    `feed` and `reset` raise ValueError as a stale iterator does.

    A leftmost_longest batch reports, over all feeds and `finish` of a stream, exactly what
    `find_leftmost_longest_batch` reports for its whole text, each match once, in chunk order then end_index
    ascending.  A match is reported by the first feed after which it starts before ``position - (longest_word - 1)``:
    from then on no later letter can change it.  `finish` reports the rest and returns those streams to their start.

    A whole_words batch reports, over all feeds and `finish` of a stream, what find_all_batch (or, leftmost_longest,
    find_leftmost_longest_batch) reports with the same whole_words for its whole text.  A find_all match is reported by
    the first feed after which at least one letter follows it, so its end_index can be the last letter of an earlier
    chunk; a leftmost_longest match by the first feed after which it starts before ``position - longest_word``.

    A leftmost_first batch is a leftmost_longest batch under the leftmost-first rule: it reports what
    `find_leftmost_first_batch` reports (with the same whole_words), at the same points.

    A batch from `Automaton.ascii_case_insensitive_stream_batch` (``ascii_case_insensitive`` True) reports what the
    batch of the same options reports, with keys and text compared ASCII case-insensitively: what the whole-batch
    method reports with ascii_case_insensitive=True for each stream's whole text.  One from
    `Automaton.case_insensitive_stream_batch` (``case_insensitive`` True) does the same with case_insensitive=True.

    A batch made with encoding="utf-8" (``encoding`` "utf-8", ``errors`` "strict" or "replace") takes UTF-8 chunks and
    reports what the batch of `str` reports for the text each stream's incremental decoder gives (see
    Automaton.stream_batch); ``pending`` tells the bytes of an unfinished letter each stream holds back."""

    def __init__(self, A: Automaton, n_streams: int, long: bool, algo: str, device: int, skip: Optional[np.ndarray] = None,
                 leftmost_longest: bool = False, words: Optional[tuple] = None, leftmost_first: bool = False,
                 fold: int = _FOLD_NONE, u8: Optional[int] = None, errors: str = "strict"):
        self._A = A
        self._fold = fold
        self.ascii_case_insensitive = fold == _FOLD_ASCII
        self.case_insensitive = fold == _FOLD_UNICODE
        self._version = A._version
        self.n_streams = n_streams
        self.long = long
        self.leftmost_longest = leftmost_longest
        self.leftmost_first = leftmost_first
        self._select = N.SELECT_FIRST if leftmost_first else N.SELECT_LONGEST
        self._words = words
        self.whole_words = words is not None
        self._algo = algo
        self._device = device
        self._pos = np.zeros(n_streams, dtype=np.int64)        # host mirror of the positions, for end_index
        self.ignore_white_space = skip is not None
        with A._gpu_lock:
            self._init_utf8(u8, errors)
            if words is not None:
                self._ss = self._native("new_words")
            elif leftmost_longest or leftmost_first:
                self._ss = self._native("new_leftmost")
            else:
                self._ss = self._native("new") if skip is None else self._native("new_skip", skip)

    def _native(self, op: str, *args):
        """Every call into the native stream batch (acb_streams_*) goes through here.
          new -> handle;  new_skip(skip set uint32) -> handle of a batch that skips those letters;  free;  reset(ids int32 or None);  positions -> int64[n_streams];
          feed(kind, data, offsets, n, stride, ids, sort) -> records (hay_id = chunk index, end_index in the chunk);
          new_leftmost -> handle of a leftmost batch (leftmost-longest or leftmost-first: self._select);
          feed_leftmost(kind, data, offsets, n, stride, ids, final) -> its chosen records, as feed's;
          new_words -> handle of a whole-word batch (leftmost or find_all, with the batch's word set);
          feed_words(kind, data, offsets, n, stride, ids, final) -> a find_all word batch's records, ordered, as feed's"""
        A = self._A
        if op == "new":
            ss = ctypes.c_void_p()
            tb, folded = self._table()
            if folded:
                N.check(A._lib.acb_streams_new_folded(tb, self.n_streams, 0, N.SELECT_LONGEST, None, -1, ctypes.byref(ss)))
            else:
                N.check(A._lib.acb_streams_new(tb, self.n_streams, int(self.long), ctypes.byref(ss)))
            return ss
        if op == "new_leftmost":
            return _new_leftmost_streams(A, self._table(), self.n_streams, self._select)
        if op == "new_words":
            return _new_word_streams(A, self._table(), self.n_streams, self.leftmost_longest or self.leftmost_first, self._words,
                                     self._select)
        if op == "new_skip":
            skip, = args
            ss = ctypes.c_void_p()
            N.check(A._lib.acb_streams_new_skip(A._ensure_table(self._device), self.n_streams, N.ptr(skip), len(skip), ctypes.byref(ss)))
            return ss
        if op in ("feed", "feed_leftmost", "feed_words"):
            return self._feed(op, *args)
        return super()._native(op, *args)

    def _feed(self, op: str, kind: str, data, offs, n: int, stride: int, ids, flag: bool, longest: Optional[int] = None) -> np.ndarray:
        """acb_streams_feed_* (flag: sort), acb_streams_feed_leftmost_* or acb_streams_feed_words_* (flag: final) -> the
        records (hay_id = chunk index, end_index in the chunk).  Overflow commits nothing: the retry is the same feed
        again, with room.  kind "letters": a decoded UTF-8 feed, data its letters (a CUDA tensor), offs their int64 CUDA
        byte offsets and longest its longest chunk in letters."""
        A = self._A
        lib, algo = A._lib, N.ALGOS[self._algo]
        ordered = op != "feed"                                  # the leftmost and word feeds order their records
        if kind == "host":
            def feed(tb, cap, found_ref):
                args = (self._ss, tb, N.ptr(data) if data.size else None, int(data.size), None if offs is None else N.ptr(offs),
                        n, stride, None if ids is None else N.ptr(ids))
                if op == "feed_leftmost":
                    return lib.acb_streams_feed_leftmost_host(*args, int(flag), None, cap, found_ref, algo)
                if op == "feed_words":
                    return lib.acb_streams_feed_words_host(*args, int(flag), None, cap, found_ref, algo)
                return lib.acb_streams_feed_host(*args, None, cap, found_ref, algo, int(flag))
            return A._host_records_on(self._table()[0], n, feed)
        import torch
        if kind == "letters":
            t, total, d_off = data, int(data.numel()), offs.data_ptr()
        else:
            t, total, d_off, longest = _stream_tensor(data, n, stride, self._device), n * stride, None, stride // A._L
        tb = self._table()[0]
        with _on_device(self._device) as stream:
            d_ids = None if ids is None else torch.from_numpy(ids).to(t.device)
            args = (self._ss, tb, t.data_ptr() if total else None, total, d_off, n, stride,
                    None if d_ids is None else d_ids.data_ptr())

            def feed(out, cap, cnt):
                if op == "feed_leftmost":
                    N.check(lib.acb_streams_feed_leftmost_device(*args, int(flag), out.data_ptr(), cap, cnt.data_ptr(), stream, algo))
                elif op == "feed_words":
                    N.check(lib.acb_streams_feed_words_device(*args, int(flag), out.data_ptr(), cap, cnt.data_ptr(), stream, algo))
                else:
                    N.check(lib.acb_streams_feed_device(*args, out.data_ptr(), cap, cnt.data_ptr(), stream, algo))
            out, found = A._device_scan(t, n, feed)
            if ordered:
                return out[:found].cpu().numpy().view(N.MATCH_DTYPE).reshape(-1)
            return A._device_records(tb, out, found, n, longest, stream, flag)

    def _stream_matches(self, rec: np.ndarray, n: int, ids32) -> Tuple[Matches, np.ndarray]:
        """A feed's records (hay_id = chunk index, end_index in the chunk) -> (Matches with stream ids and positions in
        the whole stream, the stream of every chunk)"""
        sid = np.arange(n, dtype=np.int64) if ids32 is None else ids32.astype(np.int64)
        m = Matches(rec, self._A._result_values())
        m.hay_id = sid[rec["hay_id"]]
        m.end_index = rec["end_index"].astype(np.int64) + self._pos[m.hay_id]
        return m, sid

    def _restart(self, streams) -> None:
        self._pos[streams] = 0

    def feed(self, chunks, ids=None, *, sort: bool = True) -> Matches:
        """The next chunk of some streams: chunk h continues stream ids[h] (default: stream h).  `chunks` takes the
        input forms of find_all_batch; in a list, None is an empty chunk.  Returns the matches that end inside
        these chunks (see the class); a leftmost_longest or whole_words batch returns the matches this feed settles,
        already in order (`sort` has no effect).

        A UTF-8 batch takes the UTF-8 forms of find_all_batch (a list or tuple of bytes / bytearray, None an empty
        chunk; (flat uint8, int64 byte offsets); uint8[n, stride]; a uint8 CUDA tensor [n, stride] on the batch's
        device) and reports what the batch of `str` reports for ``dec.decode(chunk)`` of each stream's incremental
        decoder.  Under errors="strict" an invalid sequence raises the UnicodeDecodeError that decoder raises for the
        first chunk (in call order) holding one -- its object is the stream's pending bytes followed by the chunk --
        and the feed changes no stream."""
        A = self._A
        with A._gpu_lock:
            self._check()
            if self._u8 is not None:
                return self._feed_utf8(chunks, ids, sort, False)
            b, lens = _stream_chunks(A, chunks)
            ids32 = self._ids(ids, b.n)
            leftmost = self.leftmost_longest or self.leftmost_first
            if leftmost or self.whole_words:
                rec = self._native("feed_leftmost" if leftmost else "feed_words", *b[:5], ids32, False)
            else:
                rec = self._native("feed", *b[:5], ids32, sort)
            m, sid = self._stream_matches(rec, b.n, ids32)
            self._pos[sid] += lens
            return m

    def finish(self, ids=None) -> Matches:
        """leftmost_longest, leftmost_first and whole_words batches: the matches streams `ids` (default: all) still hold
        back, as if their text ended here; those streams then start again at position 0 with nothing held.  Other stream
        batches of letters: ValueError.

        A UTF-8 batch first decodes each stream's pending bytes as the end of its text, as ``dec.decode(b"",
        final=True)`` does: U+FFFD under errors="replace", UnicodeDecodeError ("unexpected end of data", nothing changed)
        under "strict".  A UTF-8 find_all batch (plain, long=True or ignore_white_space=True) has a finish too: it returns
        the matches that end in those last letters, then the streams start again at position 0, as after `reset`."""
        leftmost = self.leftmost_longest or self.leftmost_first
        if not (leftmost or self.whole_words or self._u8 is not None):
            raise ValueError("finish() belongs to leftmost_longest, leftmost_first and whole_words stream batches")
        A = self._A
        with A._gpu_lock:
            self._check()
            n = self.n_streams if ids is None else len(np.asarray(ids).reshape(-1))
            if self._u8 is not None:
                ids32 = self._ids(ids, n)
                m = self._feed_utf8([b""] * n, ids32, True, True)
                if leftmost or self.whole_words:           # the final feed returned the streams to their start
                    self._restart(slice(None) if ids32 is None else ids32)
                else:                                      # a find_all feed is never final: start again as reset does
                    self._reset(ids32)
                return m
            ids32 = self._ids(ids, n)
            rec = self._native("feed_leftmost" if leftmost else "feed_words", "host", np.empty(0, np.uint8),
                               np.zeros(n + 1, np.int64), n, 0, ids32, True)
            m, sid = self._stream_matches(rec, n, ids32)
            self._restart(sid)
            return m

    def _feed_utf8(self, chunks, ids, sort: bool, final: bool) -> Matches:
        """A feed (final: the last, of finish) of a UTF-8 batch: stage and decode (_utf8_stage), the feed of this batch's
        form on the letters, then the carries committed and the positions moved"""
        f = self._utf8_stage(chunks, ids, final)
        leftmost = self.leftmost_longest or self.leftmost_first
        if leftmost or self.whole_words:
            rec = self._native("feed_leftmost" if leftmost else "feed_words", "letters", f.data, f.offsets, f.n, 0, f.ids, final,
                               f.longest)
        else:
            rec = self._native("feed", "letters", f.data, f.offsets, f.n, 0, f.ids, sort, f.longest)
        self._utf8_commit(f)
        m, sid = self._stream_matches(rec, f.n, f.ids)
        self._pos[sid] += np.diff(f.offsets.cpu().numpy()) // 4
        return m


class Replacer:
    """Result of `Automaton.replacer()`: the replacement of every key, kept on the GPU, for rewriting whole batches.

    ``replace_batch(haystacks)`` takes, per haystack, exactly the matches `find_leftmost_longest_batch` chooses, replaces
    the letters of each by its key's replacement and copies every other letter; a replacement is never scanned again.
    The replacements are a snapshot taken when the replacer is made.  A replacer belongs to the key set it was made
    for: after keys are added or removed, `replace_batch` raises ValueError as a stale iterator does.  A leftmost_first
    replacer (Automaton.replacer) takes the matches `find_leftmost_first_batch` chooses instead, in both methods."""

    def __init__(self, A: Automaton, replacements, device: int, select: int = N.SELECT_LONGEST):
        self._A = A
        self._version = A._version
        self._device = device
        self._select = select
        self.leftmost_first = select == N.SELECT_FIRST
        self._native = {}                                   # (narrow, device) -> acb_replacer*, uploaded on first use
        if replacements is None and A._store != STORE_ANY:
            raise ValueError("replacer() without replacements takes each key's value: the automaton must be STORE_ANY")
        n_ids = len(A._key_objs)
        reps = [None] * n_ids
        for kid, key in enumerate(A._key_objs):             # ids ascend in insertion order
            if key is None:
                continue
            if replacements is None:
                rep = A._values[kid]
            else:
                if key not in replacements:
                    raise KeyError(key)
                rep = replacements[key]
            reps[kid] = A._letters(rep)
        L = A._L
        empty = np.empty(0, dtype=_LETTER_DTYPE[L])
        self._tables = {False: self._layout([empty if r is None else r for r in reps], L)}
        if A._uses_narrow() and all(r is None or r.size == 0 or int(r.max()) < 256 for r in reps):
            self._tables[True] = self._layout([np.empty(0, np.uint8) if r is None else r.astype(np.uint8) for r in reps], 1)

    @staticmethod
    def _layout(letters: list, width: int) -> Tuple[np.ndarray, np.ndarray]:
        """(bytes uint8, byte offsets int64[n_ids+1]) of the replacements at `width` bytes per letter"""
        offs = np.zeros(len(letters) + 1, dtype=np.int64)
        np.cumsum(np.fromiter((a.size * width for a in letters), dtype=np.int64, count=len(letters)), out=offs[1:])
        flat = np.concatenate([np.ascontiguousarray(a, dtype=_LETTER_DTYPE[width]).view(np.uint8) for a in letters]) \
            if letters else np.empty(0, dtype=np.uint8)
        return flat, offs

    def __del__(self):
        try:
            for r in self._native.values():
                self._A._lib.acb_replacer_free(r)
            self._native = {}
        except Exception:                                   # interpreter shutdown
            pass

    def _replacer(self, tb, narrow: bool, device: int):
        """the native replacer for this table (letter width, device), uploaded on first use"""
        r = self._native.get((narrow, device))
        if r is None:
            flat, offs = self._tables[narrow]
            r = ctypes.c_void_p()
            args = (N.ptr(flat) if flat.size else None, int(flat.size), N.ptr(offs), len(offs) - 1, ctypes.byref(r))
            if self._select == N.SELECT_LONGEST:
                N.check(self._A._lib.acb_replacer_new(tb, *args))
            else:
                N.check(self._A._lib.acb_replacer_new_kind(tb, self._select, *args))
            self._native[(narrow, device)] = r
        return r

    def replace_batch(self, haystacks, *, algo: str = "auto", whole_words=False, ascii_case_insensitive: bool = False,
                      case_insensitive: bool = False, encoding: Optional[str] = None, errors: str = "strict"):
        """The batch with every leftmost-longest match replaced.  `haystacks` takes the input forms of find_all_batch;
        a list gives a list of the same item type, uint8[n, stride] or (flat, offsets) gives (flat uint8, offsets
        int64[n+1]), a CUDA tensor gives that pair as CUDA tensors computed on torch's current stream (the call
        synchronises once to size the output).  algo ("auto", "filter", "dfa") only picks the scan.  whole_words (see
        find_all_batch): replace the matches that find_leftmost_longest_batch chooses with the same option, so a key
        inside a longer word is left alone; a CUDA tensor batch then synchronises once more.  ascii_case_insensitive
        (see find_all_batch): replace the matches the find_leftmost_*_batch method of this replacer's rule chooses with
        the same option, each by the replacement of its key -- the one added first among keys that fold to the same
        text; every other letter is copied as given, in its own case.  case_insensitive (unicode flavour; see
        find_all_batch): the same with Unicode simple case folding.

        encoding and errors (see find_all_batch): UTF-8 haystacks, decoded on the GPU, and UTF-8 output, encoded on the
        GPU: exactly ``[s.encode("utf-8") for s in R.replace_batch(decoded)]`` with the same options, where decoded is
        ``[h.decode("utf-8", errors) for h in haystacks]``.  A list gives a list of bytes, uint8[n, stride] or (flat,
        offsets) gives (flat uint8, int64 byte offsets[n+1]), a CUDA tensor gives that pair as CUDA tensors.  A
        replacement that UTF-8 cannot encode (a lone surrogate) raises UnicodeEncodeError."""
        A = self._A
        with A._gpu_lock:
            if self._version != A._version:
                raise ValueError("underlaying automaton has changed, iterator is not valid anymore")
            A._require_automaton()
            if algo not in ("auto", "filter", "dfa"):
                raise ValueError(f"algo {algo!r}: replace_batch takes 'auto', 'filter' or 'dfa'")
            words = A._words(whole_words)
            fold = A._fold_arg(ascii_case_insensitive, case_insensitive=case_insensitive)
            pair = isinstance(haystacks, np.ndarray) or _is_pair(haystacks)
            u8 = A._utf8_arg(encoding, errors)
            if u8 is not None:
                self._check_utf8_replacements()
                b = A._utf8_batch(haystacks, u8, self._device, narrow_ok=True in self._tables)
                out, out_offs = self._run_utf8(b, algo, words, fold)
                if out.device.type == "cuda" and (pair or isinstance(haystacks, (list, tuple))):
                    out, out_offs = out.cpu().numpy(), out_offs.cpu().numpy()
                    if not pair:
                        raw, o = out.tobytes(), out_offs.tolist()
                        return [raw[o[i]:o[i + 1]] for i in range(len(o) - 1)]
                return out, out_offs
            batch = A._batch_input(haystacks)
            if batch.kind == "device":
                return self._run_device(batch, algo, words, fold)
            _, flat, offs, n, stride, narrow = batch
            if narrow and True not in self._tables:         # a replacement outside latin-1: 4 bytes per letter
                flat = flat.astype("<u4").view(np.uint8)
                offs = offs * 4
                narrow = False
            if offs is None:
                offs = np.arange(n + 1, dtype=np.int64) * stride
            if batch.empty:
                out, out_offs = flat[:0].copy(), np.zeros(n + 1, dtype=np.int64)
            elif fold:
                out, out_offs = self._run_host(flat, offs, n, narrow, algo, words, fold=fold)
            elif words is None:
                out, out_offs = self._run_host(flat, offs, n, narrow, algo)
            else:
                out, out_offs = self._run_host(flat, offs, n, narrow, algo, words)
            if pair:
                return out, out_offs
            return self._items(out, out_offs, narrow)

    def _check_utf8_replacements(self) -> None:
        """UnicodeEncodeError, as str.encode("utf-8") raises it, for a replacement with a lone surrogate"""
        flat, offs = self._tables[False]
        v = flat.view("<u4")
        bad = np.flatnonzero((v >= 0xD800) & (v <= 0xDFFF))
        if bad.size:
            k = int(np.searchsorted(offs, 4 * int(bad[0]), side="right")) - 1
            flat[offs[k]:offs[k + 1]].tobytes().decode("utf-32-le", "surrogatepass").encode("utf-8")

    def _run_utf8(self, b, algo: str, words: Optional[tuple], fold: int):
        """A decoded UTF-8 batch (Automaton._utf8_batch): select and rewrite as _run_device does, then encode the output
        letters to UTF-8 on the GPU (acb_utf8_encode_device); (flat, offsets) CUDA tensors.  Waits twice: for the size of
        the rewritten letters and for that of the UTF-8 output."""
        import torch
        A = self._A
        t, n = b.data, b.n
        dev = _device_of(t)
        width = 1 if b.narrow else 4
        tb = A._table_for(dev, b.narrow, fold) if n and t.numel() else None
        with _on_device(dev) as stream:
            letters, offs = t, b.offsets                    # nothing to replace: the decoded text
            if tb is not None:
                chosen, cnt, cap = A._leftmost_chosen(tb, t, n, 0, algo, stream, words, self._select, b.offsets, b.max_letters,
                                                      b.narrow)
                r = self._replacer(tb, b.narrow, dev)
                offs = torch.empty(n + 1, dtype=torch.int64, device=t.device)
                total = torch.empty(1, dtype=torch.int64, device=t.device)
                args = (r, tb, t.data_ptr(), t.numel(), b.offsets.data_ptr(), n, 0, chosen.data_ptr(), cap, cnt.data_ptr(),
                        offs.data_ptr())
                N.check(A._lib.acb_replace_device(*args, None, 0, total.data_ptr(), stream))
                m = int(total.item())
                letters = torch.empty(max(m, 16), dtype=torch.uint8, device=t.device)[:m]
                if m:
                    N.check(A._lib.acb_replace_device(*args, letters.data_ptr(), m, total.data_ptr(), stream))
            return _utf8_encode(A._lib, letters, offs, n, width, dev, stream)

    def stream_batch(self, n_streams: int, *, algo: str = "auto", device: Optional[int] = None,
                     whole_words=False, encoding: Optional[str] = None, errors: str = "strict") -> "ReplaceStream":
        """`n_streams` streams rewritten chunk by chunk (ReplaceStream.feed): over all feeds and `finish` of a stream,
        the output is exactly what `replace_batch` gives for its whole text, with the same whole_words.  Streams run at
        the automaton's full letter width (unicode: 4 bytes per letter), as every stream batch does.

        encoding="utf-8" (see Automaton.stream_batch): UTF-8 chunks in, UTF-8 out; concatenated, a stream's outputs are
        ``replace_batch([whole text], encoding="utf-8", errors=errors)``.  A replacement UTF-8 cannot encode (a lone
        surrogate) raises UnicodeEncodeError here."""
        return self._stream_batch(n_streams, algo, device, whole_words, _FOLD_NONE, encoding, errors)

    def ascii_case_insensitive_stream_batch(self, n_streams: int, *, algo: str = "auto", device: Optional[int] = None,
                                            whole_words=False, encoding: Optional[str] = None,
                                            errors: str = "strict") -> "ReplaceStream":
        """`stream_batch` with ASCII case-insensitive matching: over all feeds and `finish` of a stream, the output is
        exactly what `replace_batch` gives for its whole text with ascii_case_insensitive=True and the same whole_words.
        Each match takes the replacement of the key added first among those that fold to its text; every other letter,
        held ones included, keeps its own case.  The returned ReplaceStream has ``ascii_case_insensitive`` True.
        encoding and errors: UTF-8 chunks and output, as for stream_batch."""
        return self._stream_batch(n_streams, algo, device, whole_words, _FOLD_ASCII, encoding, errors)

    def case_insensitive_stream_batch(self, n_streams: int, *, algo: str = "auto", device: Optional[int] = None,
                                      whole_words=False, encoding: Optional[str] = None,
                                      errors: str = "strict") -> "ReplaceStream":
        """`stream_batch` with Unicode case-insensitive matching (unicode flavour): over all feeds and `finish` of a
        stream, the output is exactly what `replace_batch` gives for its whole text with case_insensitive=True and the
        same whole_words.  Each match takes the replacement of the key added first among those that fold to its text;
        every other letter, held ones included, keeps its own case.  The returned ReplaceStream has ``case_insensitive``
        True.  encoding and errors: UTF-8 chunks and output, as for stream_batch."""
        return self._stream_batch(n_streams, algo, device, whole_words, _FOLD_UNICODE, encoding, errors)

    def _stream_batch(self, n_streams: int, algo: str, device: Optional[int], whole_words, fold: int,
                      encoding: Optional[str] = None, errors: str = "strict") -> "ReplaceStream":
        """The argument check and constructor of stream_batch, ascii_case_insensitive_stream_batch and
        case_insensitive_stream_batch (fold: the fold kind)"""
        A = self._A
        with A._gpu_lock:
            if self._version != A._version:
                raise ValueError("underlaying automaton has changed, iterator is not valid anymore")
            A._require_automaton()
            u8 = A._utf8_arg(encoding, errors)
            if u8 is not None:
                self._check_utf8_replacements()
            A._fold_arg(fold == _FOLD_ASCII, case_insensitive=fold == _FOLD_UNICODE)
            n_streams = operator.index(n_streams)
            if n_streams < 0:
                raise ValueError("n_streams must not be negative")
            if algo not in ("auto", "filter", "dfa"):
                raise ValueError(f"algo {algo!r}: a replacing stream batch takes 'auto', 'filter' or 'dfa'")
            words = A._words(whole_words)
            return ReplaceStream(self, n_streams, algo, self._device if device is None else device, words, fold, u8, errors)

    def _items(self, out: np.ndarray, offs: np.ndarray, narrow: bool) -> list:
        """the output haystacks as objects of the input's type"""
        A = self._A
        b = offs.tolist()
        if A._key_type == KEY_SEQUENCE:
            v = out.view(_LETTER_DTYPE[A._L]).tolist()
            L = A._L
            return [tuple(v[b[i] // L:b[i + 1] // L]) for i in range(len(b) - 1)]
        raw = out.tobytes()
        if not A._UNICODE:
            return [raw[b[i]:b[i + 1]] for i in range(len(b) - 1)]
        if narrow:
            s = raw.decode("latin-1")
            return [s[b[i]:b[i + 1]] for i in range(len(b) - 1)]
        s = raw.decode("utf-32-le", "surrogatepass")
        return [s[b[i] // 4:b[i + 1] // 4] for i in range(len(b) - 1)]

    def _run_host(self, flat: np.ndarray, offs: np.ndarray, n: int, narrow: bool, algo: str, words: Optional[tuple] = None,
                  fold: int = _FOLD_NONE):
        """acb_replace_host (acb_replace_host_words with a word set) -> (output bytes, output offsets int64[n+1]); a
        second call when the first guess of the output size was too small (_host_bytes).  fold: on the folded table."""
        A = self._A
        tb = A._table_for(self._device, narrow, fold)
        if tb is None:                                      # no latin-1 key: nothing matches
            return flat.copy(), offs.copy()
        r = self._replacer(tb, narrow, self._device)
        out_offs = np.empty(n + 1, dtype=np.int64)
        batch = (r, tb, N.ptr(flat), int(flat.size), N.ptr(offs), n, 0)
        if words is not None:
            bits, n_bits = _word_bits(words, 1 if narrow else A._L)

        def replace(out, total_ref):
            result = (N.ALGOS[algo], N.ptr(out_offs), N.ptr(out), out.size, total_ref)
            if words is None:
                return A._lib.acb_replace_host(*batch, *result)
            return A._lib.acb_replace_host_words(*batch, N.ptr(bits) if n_bits else None, n_bits, *result)
        return _host_bytes(int(flat.size) * 5 // 4 + 4096, replace), out_offs

    def _run_device(self, batch, algo: str, words: Optional[tuple] = None, fold: int = _FOLD_NONE):
        """A CUDA tensor batch: scan, select and rewrite on torch's current stream; (flat, offsets) CUDA tensors"""
        import torch
        A = self._A
        t, n, stride = batch.data, batch.n, batch.stride
        if batch.empty:
            return torch.empty(0, dtype=torch.uint8, device=t.device), torch.zeros(n + 1, dtype=torch.int64, device=t.device)
        t = _aligned(t)
        dev = _device_of(t)
        tb = A._table_for(dev, False, fold)
        with _on_device(dev) as stream:
            chosen, cnt, cap = A._leftmost_chosen(tb, t, n, stride, algo, stream, words, self._select)
            r = self._replacer(tb, False, dev)
            out_offs = torch.empty(n + 1, dtype=torch.int64, device=t.device)
            total = torch.empty(1, dtype=torch.int64, device=t.device)
            args = (r, tb, t.data_ptr(), n * stride, None, n, stride, chosen.data_ptr(), cap, cnt.data_ptr(), out_offs.data_ptr())
            N.check(A._lib.acb_replace_device(*args, None, 0, total.data_ptr(), stream))
            m = int(total.item())                           # the one synchronisation: the size of the output
            out = torch.empty(m, dtype=torch.uint8, device=t.device)
            if m:
                N.check(A._lib.acb_replace_device(*args, out.data_ptr(), m, total.data_ptr(), stream))
        return out, out_offs


class ReplaceStream(_Streams):
    """Result of `Replacer.stream_batch()`: `n_streams` streams rewritten chunk by chunk, what they hold back kept on the
    GPU.  ``feed(chunks, ids=None)`` returns, per chunk, the stream's output that no later letter can change (every
    letter before ``position - (longest_word - 1)`` and every replacement that starts there); ``finish(ids=None)``
    returns the rest and returns those streams to their start.  Concatenated, a stream's outputs are what
    `Replacer.replace_batch` gives for its whole text.  Stale (ValueError) when the replacer is.  With whole_words, a
    stream holds back one letter more: the output before ``position - longest_word`` is released.  From
    `Replacer.ascii_case_insensitive_stream_batch` (``ascii_case_insensitive`` True), the output is what replace_batch
    gives with ascii_case_insensitive=True, released at the same points; from `Replacer.case_insensitive_stream_batch`
    (``case_insensitive`` True), what it gives with case_insensitive=True.  From a factory with encoding="utf-8", the
    chunks and the output are UTF-8 (``pending``: the bytes of an unfinished letter each stream holds back)."""

    def __init__(self, R: Replacer, n_streams: int, algo: str, device: int, words: Optional[tuple] = None, fold: int = _FOLD_NONE,
                 u8: Optional[int] = None, errors: str = "strict"):
        self._R = R
        self._fold = fold
        self.ascii_case_insensitive = fold == _FOLD_ASCII
        self.case_insensitive = fold == _FOLD_UNICODE
        self._A = R._A
        self._version = R._version
        self.n_streams = n_streams
        self._algo = algo
        self._device = device
        self._words = words
        self.whole_words = words is not None
        with self._A._gpu_lock:
            self._init_utf8(u8, errors)
            self._ss = self._native("new")

    def _native(self, op: str, *args):
        """Every call into the native batch goes through here.  new -> handle;  free;  reset(ids int32 or None);
        positions -> int64[n_streams];  feed(kind, data, offsets, n, stride, ids, final) -> (output bytes, output
        offsets int64[n+1]), numpy arrays for host chunks, CUDA tensors for a CUDA tensor or for kind "letters" (a
        decoded UTF-8 feed: data its letters, offsets their int64 CUDA byte offsets, stride 0)"""
        A = self._A
        lib = A._lib
        if op == "new":
            if self._words is not None:
                return _new_word_streams(A, self._table(), self.n_streams, True, self._words, self._R._select)
            return _new_leftmost_streams(A, self._table(), self.n_streams, self._R._select)
        if op != "feed":
            return super()._native(op, *args)
        kind, data, offs, n, stride, ids, final = args
        tb = self._table()[0]
        r = self._R._replacer(tb, False, self._device)
        algo = N.ALGOS[self._algo]
        held = n * max(int(lib.acb_trie_longest_word(A._trie)) - 1 + self.whole_words, 0) * A._L   # at most what is held back
        if kind == "host":
            size = int(data.size)
            out_offs = np.empty(n + 1, dtype=np.int64)
            out = _host_bytes((size + held) * 5 // 4 + 4096, lambda out, total_ref: lib.acb_streams_replace_host(
                self._ss, r, tb, N.ptr(data) if size else None, size, None if offs is None else N.ptr(offs), n, stride,
                None if ids is None else N.ptr(ids), int(final), algo, N.ptr(out_offs), N.ptr(out), out.size, total_ref))
            return out, out_offs
        import torch
        if kind == "letters":
            t, size, d_off = data, int(data.numel()), offs.data_ptr()
        else:
            t, size, d_off = _stream_tensor(data, n, stride, self._device), n * stride, None
        with _on_device(self._device) as stream:
            d_ids = None if ids is None else torch.from_numpy(ids).to(t.device)
            out_offs = torch.empty(n + 1, dtype=torch.int64, device=t.device)
            total = torch.empty(1, dtype=torch.int64, device=t.device)
            cap = (size + held) * 5 // 4 + 4096
            for retry in (False, True):
                out = torch.empty(cap, dtype=torch.uint8, device=t.device)
                N.check(lib.acb_streams_replace_device(self._ss, r, tb, t.data_ptr() if size else None, size,
                                                       d_off, n, stride, None if d_ids is None else d_ids.data_ptr(),
                                                       int(final), out_offs.data_ptr(), out.data_ptr(), cap,
                                                       total.data_ptr(), stream, algo))
                m = int(total.item())                       # the size of the output
                if m <= cap:
                    return out[:m], out_offs
                if retry:
                    raise N.NativeError(f"{m} output bytes after a retry with room for {cap}")
                cap = m                                     # nothing was committed: the same feed again, with room

    def feed(self, chunks, ids=None):
        """The next chunk of some streams (chunk h continues stream ids[h], default stream h), in the input forms of
        find_all_batch; in a list, None is an empty chunk.  Returns the output each chunk releases: a list gives a list
        of the same item type, uint8[n, stride] or (flat, offsets) gives (flat uint8, offsets int64[n+1]), a CUDA
        tensor gives that pair as CUDA tensors computed on torch's current stream.

        A UTF-8 batch takes the UTF-8 forms of StreamBatch.feed and returns UTF-8: a list of bytes for a list, (flat
        uint8, int64 byte offsets[n+1]) for an array or pair, that pair as CUDA tensors for a CUDA tensor.  Errors are
        raised as by StreamBatch.feed, and a feed that raises changes no stream."""
        A = self._A
        with A._gpu_lock:
            self._check()
            if self._u8 is not None:
                form = "pair" if isinstance(chunks, np.ndarray) or _is_pair(chunks) else \
                    "list" if isinstance(chunks, (list, tuple)) else "device"
                return self._feed_utf8(chunks, ids, False, form)
            b, _ = _stream_chunks(A, chunks)
            out, offs = self._native("feed", *b[:5], self._ids(ids, b.n), False)
            if isinstance(chunks, np.ndarray) or _is_pair(chunks) or b.kind == "device":
                return out, offs
            return self._R._items(out, offs, False)

    def finish(self, ids=None) -> list:
        """The output streams `ids` (default: all) still hold back, one item of the haystack type per id; those streams
        then start again at position 0 with nothing held.  A UTF-8 batch decodes each stream's pending bytes as the end
        of its text first (see StreamBatch.finish) and returns a list of bytes."""
        A = self._A
        with A._gpu_lock:
            self._check()
            n = self.n_streams if ids is None else len(np.asarray(ids).reshape(-1))
            if self._u8 is not None:
                return self._feed_utf8([b""] * n, self._ids(ids, n), True, "list")
            out, offs = self._native("feed", "host", np.empty(0, np.uint8), np.zeros(n + 1, np.int64), n, 0, self._ids(ids, n), True)
            return self._R._items(out, offs, False)


    def _feed_utf8(self, chunks, ids, final: bool, form: str):
        """A replacing feed of a UTF-8 batch: stage and decode (_utf8_stage), rewrite, commit the carries, encode the
        released letters to UTF-8 on the GPU; form "list" (a list of bytes), "pair" (numpy flat and offsets) or "device"
        (CUDA tensors)"""
        f = self._utf8_stage(chunks, ids, final)
        letters, offs = self._native("feed", "letters", f.data, f.offsets, f.n, 0, f.ids, final)
        self._utf8_commit(f)
        with _on_device(self._device) as stream:
            out, offs = _utf8_encode(self._A._lib, letters, offs, f.n, 4, self._device, stream)
        if form == "device":
            return out, offs
        out, offs = out.cpu().numpy(), offs.cpu().numpy()
        if form == "pair":
            return out, offs
        raw, o = out.tobytes(), offs.tolist()
        return [raw[o[i]:o[i + 1]] for i in range(f.n)]


class AutomatonSearchIter:
    """Result of `Automaton.iter()` (src/AutomatonSearchIter.c).  Matches of the current chunk are
    produced by one GPU scan when the chunk is installed; `set()` continues the stream."""

    def __init__(self, A: Automaton, letters: np.ndarray, start: int, end: int, ignore_ws: bool):
        self._A = A
        self._version = A._version                                  # :84
        self._ignore_ws = ignore_ws
        self._shift = 0
        self._hist = letters[:0]                                    # consumed letters that can still start a match
        self._pending: list = []
        self._install(letters, start, end)
        self._index = start - 1                                     # :123

    def _install(self, letters, start, end):
        """Scan letters[start:end] as the continuation of the stream."""
        A = self._A
        seg = letters[start:end]
        if self._ignore_ws:
            keep = ~_space_mask(seg, not A._UNICODE and A._key_type == KEY_STRING)
            pos = np.nonzero(keep)[0] + start                       # original index of every kept letter
            seg = seg[keep]
        else:
            pos = None
        nh = len(self._hist)
        if nh and self._hist.dtype != seg.dtype:                    # a narrow (latin-1) chunk after a wide one or vice versa
            wide = np.dtype("<u4")
            self._hist = self._hist.astype(wide)
            seg = seg.astype(wide)
        data = np.concatenate([self._hist, seg]) if nh else seg
        rec = A._scan_one(data) if len(data) else np.empty(0, dtype=N.MATCH_DTYPE)
        ends = rec["end_index"]
        sel = ends >= nh                                            # matches ending inside the history were reported before
        ends = ends[sel] - nh
        kids = rec["key_id"][sel]
        idx = pos[ends] if pos is not None else ends + start
        self._matches = list(zip(idx.tolist(), kids.tolist()))
        self._cursor = 0
        self._seg = seg
        self._seg_pos = pos
        self._start = start
        self._end = end

    def __iter__(self):
        return self

    def __next__(self):
        A = self._A
        if self._version != A._version:
            raise ValueError("underlaying automaton has changed, iterator is not valid anymore")   # :247-250
        if self._pending:                                           # outputs left over from before set()
            k = self._pending.pop(0)
            return (self._index + self._shift, A._values[k])
        if self._cursor < len(self._matches):
            i, k = self._matches[self._cursor]
            self._cursor += 1
            self._index = i
            return (i + self._shift, A._values[k])
        self._index = max(self._end, self._index + 1)               # where the reference's index stops
        raise StopIteration

    def set(self, *args):
        """src/AutomatonSearchIter.c:303-368: set(string, reset=False)."""
        if not args:
            raise IndexError("tuple index out of range")
        A = self._A
        letters = A._hay_letters(args[0])
        reset = bool(args[1]) if len(args) > 1 else False
        if reset:
            self._hist = letters[:0]
            self._shift = 0
            self._pending = []
        else:
            # letters consumed so far = everything up to and including the current index
            consumed_upto = self._index
            if self._seg_pos is not None:
                ncons = int(np.searchsorted(self._seg_pos, consumed_upto, side="right"))
            else:
                ncons = min(max(consumed_upto - self._start + 1, 0), len(self._seg))
            keep = max(int(A._lib.acb_trie_longest_word(A._trie)) - 1, 0)
            old = self._seg[:ncons]
            if len(self._hist) and self._hist.dtype != old.dtype:
                old = old.astype(self._hist.dtype) if self._hist.dtype.itemsize > old.dtype.itemsize else old
                if self._hist.dtype != old.dtype:
                    self._hist = self._hist.astype(old.dtype)
            hist = np.concatenate([self._hist, old])
            self._hist = hist[max(len(hist) - keep, 0):] if keep else hist[:0]
            # outputs of the current position not yet returned stay pending (iter->output survives set())
            if not self._pending:
                self._pending = [k for i, k in self._matches[self._cursor:] if i == self._index]
            self._shift += self._index if self._index >= 0 else 0   # :344-352
        self._install(letters, 0, len(letters))
        self._index = -1                                            # :354
        return None


class AutomatonSearchIterLong:
    """Result of `Automaton.iter_long()` (src/AutomatonSearchIterLong.c).  The reference walks lazily; here every
    chunk is scanned once on the GPU (ACB_ALGO_LONG replays the reference's state machine) when it is handed
    over, and `__next__` pays the matches out.  What `set()` must carry over is reconstructed from how far the
    caller had iterated:

    * the walk restarts from the root after every match it returns (:104-112), so once a match of the current
      chunk has been returned and the chunk is not exhausted, the carried state is the root;
    * after exhaustion it is the node the walk has reached -- the kernel hands that state id back
      (`acb_table_get_long_state`) and the next chunk starts in it (`acb_table_set_long_state`): only the new
      chunk is uploaded and scanned, whatever the length of the stream (the first version re-scanned the letters
      since the last restart point, which grows without bound on a stream without matches);
    * a chunk of which nothing was consumed leaves the state it was entered with.
    """

    def __init__(self, A: Automaton, letters: np.ndarray, start: int, end: int):
        self._A = A
        self._version = A._version
        self._shift = 0
        self._state = 0                                       # iter->state, as a state id of the flattened automaton
        self._load(letters, start, end)

    def _load(self, letters: np.ndarray, start: int, end: int) -> None:
        seg = letters[start:end] if end > start else letters[:0]
        A = self._A
        self._state_in = self._state if self._version == A._version else 0
        if len(seg):
            rec = A._scan_one(seg, algo="long", long_state=self._state_in)
            self._state_out = A._long_state_out
        else:
            rec = np.empty(0, dtype=N.MATCH_DTYPE)
            self._state_out = self._state_in
        ends = (rec["end_index"].astype(np.int64) + start).tolist()
        self._matches = list(zip(ends, rec["key_id"].tolist()))
        self._cursor = 0
        self._seg = seg
        self._start, self._end = start, end
        self._index = start - 1                               # :34
        self._exhausted = False

    def __iter__(self):
        return self

    def __next__(self):
        if self._version != self._A._version:
            raise ValueError("underlaying automaton has changed, iterator is not valid anymore")
        if self._cursor >= len(self._matches):
            self._index += 1                                  # :115, executed on every call
            if self._index < self._end:
                self._index = self._end
            self._exhausted = True
            raise StopIteration
        i, k = self._matches[self._cursor]
        self._cursor += 1
        self._index = i                                       # :108
        return (i + self._shift, self._A._values[k])

    def set(self, *args):
        """set(string, reset=False), :156-212: continue with the next chunk, keeping the walk's state and adding
        the current index to the offset of the reported positions -- unless `reset`."""
        if len(args) < 1:
            raise IndexError("tuple index out of range")
        letters = self._A._letters(args[0], required=True)
        reset = bool(args[1]) if len(args) >= 2 else False
        if reset:
            self._shift = 0
            self._state = 0
        else:
            if self._index >= 0:
                self._shift += self._index                    # :195-196
            if self._exhausted:
                self._state = self._state_out                 # the whole chunk was walked: the state it ended in
            elif self._cursor:
                self._state = 0                               # a match was just returned: the walk is at the root
            else:
                self._state = self._state_in                  # nothing of the old chunk was consumed
        self._load(letters, 0, len(letters))
        self._index = -1                                      # :198


# ---------------------------------------------------------------------- helpers
def _parse_start_end(args, i_start, i_end, lo, hi):
    """src/utils.c:293-359 (negative end is len-1+end, sic -- SURVEY A3)."""
    start, end = lo, hi
    if len(args) <= i_start:
        return start, end
    start = operator.index(args[i_start])
    if start < 0:
        start = hi + start
    if start < lo or start >= hi:
        raise IndexError(f"start index not in range {lo}..{hi}")
    if len(args) <= i_end:
        return start, end
    end = operator.index(args[i_end])
    if end < 0:
        end = hi - 1 + end
    if end < lo or end > hi:
        raise IndexError(f"end index not in range {lo}..{hi}")
    return start, end


def _take_records(lib, tb, found: int) -> np.ndarray:
    """The records of the last host-buffer call on `tb`, without a copy: they stay in the pinned buffer the D2H landed
    in, which returns to the library's pool when the last array that views it is gone (_PinnedRecords.__del__)."""
    ptr, n, room = ctypes.c_void_p(), ctypes.c_int64(0), ctypes.c_int64(0)
    N.check(lib.acb_take_records(tb, ctypes.byref(ptr), ctypes.byref(n), ctypes.byref(room)))
    if not ptr.value or n.value != found:
        raise N.NativeError("acb_take_records: no records to take")
    return np.asarray(_PinnedRecords(lib, ptr.value, n.value, room.value))


class _Utf8Batch(NamedTuple):
    """A UTF-8 batch decoded on the GPU (Automaton._utf8_batch): data, its letters (1-D uint8 CUDA tensor, 16-byte
    aligned); offsets, their int64 CUDA byte offsets [n + 1]; max_letters, the longest haystack; narrow: 1 byte per
    letter."""
    data: Any
    offsets: Any
    n: int
    max_letters: int
    narrow: bool


class _Utf8Feed(NamedTuple):
    """A UTF-8 feed staged and decoded on the GPU (_Streams._utf8_stage): data, its 4-byte letters (1-D uint8 CUDA
    tensor, 16-byte aligned); offsets, their int64 CUDA byte offsets [n + 1]; longest, the longest chunk in letters;
    ids, the stream ids (int32 or None) and d_ids, their CUDA copy."""
    data: Any
    offsets: Any
    n: int
    longest: int
    ids: Optional[np.ndarray]
    d_ids: Any


def _utf8_error(t, host, stride: int, start: int, end: int) -> UnicodeDecodeError:
    """CPython's UnicodeDecodeError for the invalid sequence at bytes [start, end) of a UTF-8 batch: the haystack that
    holds it, and the sequence's place in it"""
    if host is not None and host[1] is not None:
        flat, offs = host
        h = int(np.searchsorted(offs, start, side="right")) - 1
        hs, he = int(offs[h]), int(offs[h + 1])
    else:
        hs = start // stride * stride
        he = hs + stride
    hay = bytes((host[0][hs:he] if host is not None else t[hs:he].cpu().numpy()).tobytes())
    return _decode_error(hay, start - hs, end - hs)


def _decode_error(hay: bytes, start: int, end: int) -> UnicodeDecodeError:
    """CPython's UnicodeDecodeError for the invalid sequence at bytes [start, end) of hay"""
    if not 0xC2 <= hay[start] <= 0xF4:
        reason = "invalid start byte"
    elif end == len(hay):
        reason = "unexpected end of data"
    else:
        reason = "invalid continuation byte"
    return UnicodeDecodeError("utf-8", hay, start, end, reason)


def _utf8_encode(lib, letters, offs, n: int, width: int, dev: int, stream):
    """letters of `width` bytes (a CUDA tensor) at the int64 CUDA byte offsets offs [n + 1] -> their UTF-8, encoded on
    the GPU (acb_utf8_encode_device) on `stream`: (flat uint8, int64 byte offsets [n + 1]) CUDA tensors.  Waits once,
    for the size."""
    import torch
    need = ctypes.c_int64(0)
    N.check(lib.acb_utf8_work_bytes(0, n, ctypes.byref(need)))
    work = torch.empty(int(need.value), dtype=torch.uint8, device=letters.device)
    cap = letters.numel() // width * (2 if width == 1 else 4)     # the most UTF-8 bytes a letter takes at this width
    out = torch.empty(max(cap, 1), dtype=torch.uint8, device=letters.device)
    out_offs = torch.empty(n + 1, dtype=torch.int64, device=letters.device)
    total = torch.empty(1, dtype=torch.int64, device=letters.device)
    N.check(lib.acb_utf8_encode_device(dev, letters.data_ptr() if letters.numel() else None, letters.numel(),
                                       offs.data_ptr(), n, width, work.data_ptr(), work.numel(), out.data_ptr(),
                                       cap, out_offs.data_ptr(), total.data_ptr(), stream))
    return out[:int(total.item())], out_offs


class _Batch(NamedTuple):
    """A batch as _batch_input lays it out.  kind "device": data is the CUDA tensor [n, stride] itself; kind "host": data
    is the flat uint8 buffer and offsets its int64 byte offsets, or None for rows of a fixed stride (else stride is 0).
    narrow: the buffer holds the 1-byte letters of the latin-1 automaton."""
    kind: str
    data: Any
    offsets: Optional[np.ndarray]
    n: int
    stride: int
    narrow: bool

    @property
    def empty(self) -> bool:
        """no haystack or no letter at all: nothing can match"""
        return self.n == 0 or (self.stride if self.kind == "device" else self.data.size) == 0


def _is_pair(x) -> bool:
    """x is the (flat, offsets) input form of the batch methods"""
    return isinstance(x, tuple) and len(x) == 2 and isinstance(x[0], np.ndarray) and isinstance(x[1], np.ndarray)


def _stream_chunks(A: Automaton, chunks):
    """A stream feed's chunks in the input forms of find_all_batch (in a list, None is an empty chunk) at the
    automaton's full letter width -> (_Batch, letters per chunk int64[n])"""
    if isinstance(chunks, list) or (isinstance(chunks, tuple) and not _is_pair(chunks)):
        empty = () if A._key_type == KEY_SEQUENCE else ("" if A._UNICODE else b"")
        chunks = [empty if c is None else c for c in chunks]
    b = A._batch_input(chunks, narrow_ok=False)
    if b.kind == "device":
        return b, np.full(b.n, b.stride // A._L, dtype=np.int64)
    return b, (np.diff(b.offsets) if b.offsets is not None else np.full(b.n, b.stride, dtype=np.int64)) // A._L


def _stream_tensor(t, n: int, stride: int, device: int):
    """a CUDA tensor of chunks for a stream batch on `device`, 16-byte aligned"""
    dev = _device_of(t)
    if dev != device:
        raise ValueError(f"chunks on cuda:{dev} for a stream batch on cuda:{device}")
    return _aligned(t) if n and stride else t


def _device_of(t) -> int:
    """the index of the CUDA device a tensor lives on"""
    import torch
    return t.device.index if t.device.index is not None else torch.cuda.current_device()


@contextlib.contextmanager
def _on_device(dev: int):
    """CUDA device `dev` made current for the block, which gets torch's current stream on it (a cudaStream_t)"""
    import torch
    with torch.cuda.device(dev):
        yield torch.cuda.current_stream().cuda_stream


def _host_bytes(cap: int, call) -> np.ndarray:
    """The output of one host call that writes bytes: call(out, total_ref) writes into out, a fresh uint8[cap], and
    returns its status.  On ACB_EOVERFLOW it runs once more with room for the exact total; a second overflow raises."""
    total = ctypes.c_int64(0)
    out = np.empty(cap, dtype=np.uint8)
    rc = call(out, ctypes.byref(total))
    if rc == N.ACB_EOVERFLOW:
        out = np.empty(int(total.value), dtype=np.uint8)
        rc = call(out, ctypes.byref(total))
    N.check(rc)
    return out[:total.value]


def _new_leftmost_streams(A: Automaton, table, n_streams: int, select: int = N.SELECT_LONGEST):
    """a leftmost stream batch on table = (tb, folded) (_Streams._table)"""
    ss = ctypes.c_void_p()
    tb, folded = table
    if folded:
        N.check(A._lib.acb_streams_new_folded(tb, n_streams, 1, select, None, -1, ctypes.byref(ss)))
    elif select == N.SELECT_LONGEST:
        N.check(A._lib.acb_streams_new_leftmost(tb, n_streams, ctypes.byref(ss)))
    else:
        N.check(A._lib.acb_streams_new_leftmost_kind(tb, n_streams, select, None, -1, ctypes.byref(ss)))
    return ss


def _new_word_streams(A: Automaton, table, n_streams: int, leftmost: bool, words: tuple, select: int = N.SELECT_LONGEST):
    """a whole-word stream batch (acb_streams_new_words; acb_streams_new_leftmost_kind for leftmost-first;
    acb_streams_new_folded on a folded table) on table = (tb, folded) (_Streams._table) with the word set at the
    streams' full letter width"""
    bits, n_bits = _word_bits(words, A._L)
    ss = ctypes.c_void_p()
    tb, folded = table
    if folded:
        N.check(A._lib.acb_streams_new_folded(tb, n_streams, int(leftmost), select, N.ptr(bits) if n_bits else None, n_bits,
                                              ctypes.byref(ss)))
    elif leftmost and select != N.SELECT_LONGEST:
        N.check(A._lib.acb_streams_new_leftmost_kind(tb, n_streams, select, N.ptr(bits) if n_bits else None, n_bits,
                                                     ctypes.byref(ss)))
    else:
        N.check(A._lib.acb_streams_new_words(tb, n_streams, int(leftmost), N.ptr(bits) if n_bits else None, n_bits,
                                             ctypes.byref(ss)))
    return ss


def _aligned(t):
    """A device batch whose data starts on a 16-byte boundary, as the scan's TMA bulk copies need: `t` itself, or for
    a view that starts elsewhere (e.g. d[1:] of a [n, 7] tensor) a copy in fresh storage on the same device, made on
    the current stream."""
    return t if t.data_ptr() % 16 == 0 else t.clone()


def _default_device() -> int:
    try:
        import torch
        if torch.cuda.is_available():
            return torch.cuda.current_device()
    except Exception:
        pass
    return 0


def _rebuild(unicode_flavour, args):
    from . import flavour
    return flavour("unicode" if unicode_flavour else "bytes").Automaton(*args)


def load(*args):
    """ahocorasick.load(path, deserializer) for the package's default flavour (src/custompickle/load/)."""
    import pyahocorasick_b200 as pkg
    from . import serialize
    return serialize.load(pkg.Automaton, *args)
