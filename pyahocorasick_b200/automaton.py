"""`Automaton` -- the reference's Python surface (src/Automaton.c:1204-1256) on top of the
H100 C ABI (include/acb200.h).

Host side (this file + csrc/acb_host.cpp): keys, values, state machine EMPTY -> TRIE ->
AHOCORASICK, argument parsing and error behaviour of the reference.
Device side (csrc/acb_device.cu): every search -- `iter`, `find_all`, and the batch entry
`find_all_batch` -- runs on the GPU; there is no CPU search path in this package.

Reference semantics are cited as file:line relative to /root/reference.
"""
from __future__ import annotations

import ctypes
import functools
import os
import operator
import pickle
import threading
from typing import Any, Iterable, List, Optional, Sequence, Tuple

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


_libc = ctypes.CDLL(None)
_libc.iswspace.argtypes = [ctypes.c_uint]
_libc.iswspace.restype = ctypes.c_int


def _space_mask(letters: np.ndarray, bytes_flavour: bool) -> np.ndarray:
    """iswspace() of every letter, as the reference evaluates it (src/AutomatonSearchIter.c:270-274).
    The bytes flavour widens through a signed char first (src/utils.c:199-202)."""
    if letters.size == 0:
        return np.zeros(0, dtype=bool)
    vals = letters.astype(np.uint32)
    if bytes_flavour and letters.dtype == np.uint8:
        vals = letters.astype(np.int8).astype(np.int16).astype(np.uint16).astype(np.uint32)
    uniq = np.unique(vals)
    spaces = np.array([u for u in uniq.tolist() if _libc.iswspace(u)], dtype=np.uint32)
    return np.isin(vals, spaces)


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
    (hay_id, then end_index ascending, then longest key first)."""

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
        self._version = 0
        self._table = None                # acb_table* (device), created lazily
        self._table_device = None
        # unicode flavour only: a second, 1-byte-per-letter automaton over the keys that are pure latin-1,
        # built lazily and used whenever a haystack is latin-1 too (4x fewer bytes to move and scan)
        self._narrow_trie = None
        self._narrow_table = None
        self._narrow_device = None
        self._narrow_empty = False
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
        self._version += 1
        self._drop_table()

    # keys / values / items (src/AutomatonItemsIter.c) -- host-only enumeration
    def _select(self, args):
        prefix = None
        wildcard = None
        how = MATCH_EXACT_LENGTH
        if len(args) >= 1 and args[0] is not None:
            prefix = args[0]
            self._letters(prefix)
        if len(args) >= 2 and args[1] is not None:
            wildcard = args[1]
            wl = self._letters(wildcard)
            if len(wl) != 1:
                raise ValueError("Wildcard must be a single character.")
        if len(args) >= 3:
            how = args[2]
            if how not in (MATCH_EXACT_LENGTH, MATCH_AT_MOST_PREFIX, MATCH_AT_LEAST_PREFIX):
                raise ValueError("The optional how third argument must be one of: "
                                 "MATCH_EXACT_LENGTH, MATCH_AT_LEAST_PREFIX or MATCH_AT_LEAST_PREFIX")
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
            w = None if wildcard is None else int(self._letters(wildcard)[0])
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
        fv = N.FlatView()
        trie = self._trie
        if narrow:
            trie = self._narrow_host()
            if trie is None:
                return None
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
                   long_state: Optional[int] = None) -> np.ndarray:
        """flat uint8 buffer (+ int64 byte offsets or a fixed stride) -> sorted match records.
        narrow=True: the buffer holds 1-byte letters of a unicode-flavour automaton (latin-1 path).
        long_state (algo "long", one haystack): the state the walk starts in; the state it ends in is left in
        self._long_state_out (iter_long streaming, acb_table_set_long_state / acb_table_get_long_state)."""
        if narrow:
            core = self._ensure_narrow(device)
            if core is None:
                return np.empty(0, dtype=N.MATCH_DTYPE)
            tb = core[1]
        else:
            tb = self._ensure_table(device)
        total = int(flat.size)
        cap = max(self._match_cap, 1 << 12, 2 * n_hay)        # device-side capacity; grown on overflow
        found = ctypes.c_int64(0)
        while True:
            if long_state is not None:
                N.check(self._lib.acb_table_set_long_state(tb, int(long_state)))      # one shot: again before a retry
            rc = self._lib.acb_scan_host(tb, N.ptr(flat) if total else None, total,
                                         N.ptr(offsets) if offsets is not None else None, n_hay, stride_bytes,
                                         None, cap, ctypes.byref(found), N.ALGOS[algo], 1 if sort else 0)
            if rc == N.ACB_EOVERFLOW:
                cap = int(found.value) + 1024
                self._match_cap = cap
                continue
            N.check(rc)
            if long_state is not None:
                st = ctypes.c_int32(0)
                N.check(self._lib.acb_table_get_long_state(tb, ctypes.byref(st)))
                self._long_state_out = int(st.value)
            if not found.value:
                return np.empty(0, dtype=N.MATCH_DTYPE)
            # no copy: the records stay in the pinned buffer the D2H landed in; it returns to the library's pool
            # when the last array that views it is gone (_PinnedRecords.__del__)
            ptr, n, room = ctypes.c_void_p(), ctypes.c_int64(0), ctypes.c_int64(0)
            N.check(self._lib.acb_take_records(tb, ctypes.byref(ptr), ctypes.byref(n), ctypes.byref(room)))
            if not ptr.value or n.value != found.value:
                raise N.NativeError("acb_take_records: no records to take")
            return np.asarray(_PinnedRecords(self._lib, ptr.value, n.value, room.value))

    @_locked
    def _scan_device_tensor(self, t, algo: str, sort: bool) -> np.ndarray:
        """Batch already resident in HBM: a C-contiguous uint8 torch CUDA tensor [n, stride].  No host copy of
        the haystacks; the scan runs on torch's current stream, only the records come back."""
        import torch
        if t.dtype != torch.uint8 or t.dim() != 2 or not t.is_contiguous():
            raise TypeError("device batches must be 2-D contiguous uint8 tensors [n_haystacks, stride_bytes]")
        n, stride = int(t.shape[0]), int(t.shape[1])
        if stride % self._L:
            raise ValueError("row length must be a multiple of the letter width")
        if n == 0 or stride == 0:
            return np.empty(0, dtype=N.MATCH_DTYPE)
        dev = t.device.index if t.device.index is not None else torch.cuda.current_device()
        tb = self._ensure_table(dev)
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream().cuda_stream
            cnt = torch.zeros(1, dtype=torch.int64, device=t.device)
            cap = max(self._match_cap, 1 << 12, 2 * n)
            while True:
                out = torch.empty((cap, 3), dtype=torch.int32, device=t.device)
                cnt.zero_()
                N.check(self._lib.acb_scan_device(tb, t.data_ptr(), n * stride, None, n, stride, out.data_ptr(), cap,
                                                  cnt.data_ptr(), stream, N.ALGOS[algo]))
                found = int(cnt.item())
                if found > cap:
                    cap = self._match_cap = found + 1024
                    continue
                break
            if sort and found > 1:
                rc = self._lib.acb_sort_matches_device(tb, out.data_ptr(), found, n, stride // self._L, stream)
                if rc == N.ACB_ERANGE:
                    sort_on_host = True
                else:
                    N.check(rc)
                    sort_on_host = False
            else:
                sort_on_host = False
            rec = out[:found].cpu().numpy().view(N.MATCH_DTYPE).reshape(-1)
        if sort_on_host:
            kl = np.asarray(self.flat()["key_len"])
            rec = rec[np.lexsort((-kl[rec["key_id"]], rec["end_index"], rec["hay_id"]))]
        return rec

    def _scan_one(self, letters: np.ndarray, algo: str = "auto", long_state: Optional[int] = None) -> np.ndarray:
        narrow = self._uses_narrow() and letters.dtype == np.uint8 and algo != "long"
        if self._uses_narrow() and letters.dtype == np.uint8 and not narrow:
            letters = letters.astype("<u4")                  # iter_long never runs on the latin-1 automaton
        flat = np.ascontiguousarray(letters).view(np.uint8)
        if flat.size == 0:
            return np.empty(0, dtype=N.MATCH_DTYPE)
        if narrow:
            return self._scan_flat(flat, None, 1, int(flat.size), algo=algo, narrow=True)
        if long_state is not None:
            return self._scan_flat(flat, None, 1, int(flat.size), algo=algo, long_state=long_state)
        return self._scan_flat(flat, None, 1, int(flat.size), algo=algo)

    def _require_automaton(self):
        if self.kind != AHOCORASICK:
            raise AttributeError("Not an Aho-Corasick automaton yet: call add_word to add some keys and call "
                                 "make_automaton to convert the trie to an automaton.")

    # ------------------------------------------------------------------ search API of the reference
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

    def find_long_batch(self, haystacks, *, sort: bool = True, device: Optional[int] = None) -> "Matches":
        """iter_long() over a whole batch (same input forms and result type as find_all_batch)."""
        return self.find_all_batch(haystacks, algo="long", sort=sort, device=device)

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
    def find_all_batch(self, haystacks, *, algo: str = "auto", sort: bool = True, device: Optional[int] = None) -> Matches:
        """Search a whole batch on the GPU.

        haystacks: a sequence of bytes / str / tuple objects (as `iter` accepts), or a 2-D
        C-contiguous uint8 array [n, stride] (bytes flavour: one haystack per row), or a pair
        (flat uint8 array, int64 byte offsets of length n+1), or a 2-D contiguous uint8 torch CUDA
        tensor [n, stride] that already lives in HBM (no host copy of the batch).

        Equivalent to ``[(h, e, v) for h, hay in enumerate(haystacks) for e, v in A.iter(hay)]``
        of the reference, returned as arrays.
        """
        self._require_automaton()
        L = self._L
        if type(haystacks).__module__.startswith("torch") and getattr(haystacks, "is_cuda", False):
            return Matches(self._scan_device_tensor(haystacks, algo, sort), self._values)
        if isinstance(haystacks, np.ndarray):
            if haystacks.dtype != np.uint8 or haystacks.ndim != 2 or not haystacks.flags.c_contiguous:
                raise TypeError("array batches must be 2-D C-contiguous uint8 [n_haystacks, stride_bytes]")
            n, stride = haystacks.shape
            if stride % L:
                raise ValueError("row length must be a multiple of the letter width")
            rec = self._scan_flat(haystacks.reshape(-1), None, n, stride, algo=algo, sort=sort, device=device) if n and stride else np.empty(0, dtype=N.MATCH_DTYPE)
            return Matches(rec, self._values)
        if isinstance(haystacks, tuple) and len(haystacks) == 2 and isinstance(haystacks[0], np.ndarray) and isinstance(haystacks[1], np.ndarray):
            flat = np.ascontiguousarray(haystacks[0], dtype=np.uint8).reshape(-1)
            offs = np.ascontiguousarray(haystacks[1], dtype=np.int64)
            if offs.ndim != 1 or len(offs) < 1 or offs[0] != 0 or offs[-1] != flat.size or np.any(np.diff(offs) < 0) or np.any(offs % L):
                raise ValueError("offsets must be non-decreasing multiples of the letter width, start at 0 and end at len(flat)")
            n = len(offs) - 1
            rec = self._scan_flat(flat, offs, n, 0, algo=algo, sort=sort, device=device) if n and flat.size else np.empty(0, dtype=N.MATCH_DTYPE)
            return Matches(rec, self._values)
        # the latin-1 automaton finds exactly the matches of a latin-1 haystack -- all of them.  iter_long's walk is
        # different: which match it keeps depends on the whole trie (a non-latin-1 key whose prefix is latin-1 adds
        # nodes the walk passes through, src/AutomatonSearchIterLong.c:118-126), so it always runs on the full one
        if not self._UNICODE and self._key_type == KEY_STRING and isinstance(haystacks, (list, tuple)) and haystacks \
                and set(map(type, haystacks)) == {bytes}:       # C-level pass, 3 x faster than a generator with all()
            # the common drop-in input, a list of bytes objects: one join instead of an array per haystack
            n = len(haystacks)
            offs = np.zeros(n + 1, dtype=np.int64)
            np.cumsum(np.fromiter(map(len, haystacks), dtype=np.int64, count=n), out=offs[1:])
            flat = np.frombuffer(b"".join(haystacks), dtype=np.uint8)
            if not flat.size:
                return Matches(np.empty(0, dtype=N.MATCH_DTYPE), self._values)
            return Matches(self._scan_flat(flat, offs, n, 0, algo=algo, sort=sort, device=device), self._values)
        get = self._letters if algo == "long" else self._hay_letters
        letters = [get(h, required=True) for h in haystacks]
        narrow = self._uses_narrow() and len(letters) > 0 and all(a.dtype == np.uint8 for a in letters)
        if self._uses_narrow() and not narrow:                   # mixed batch: everything at 4 bytes per letter
            letters = [a.astype("<u4") if a.dtype == np.uint8 else a for a in letters]
        parts = [np.ascontiguousarray(a).view(np.uint8) for a in letters]
        n = len(parts)
        lens = np.fromiter((p.size for p in parts), dtype=np.int64, count=n)
        offs = np.zeros(n + 1, dtype=np.int64)
        np.cumsum(lens, out=offs[1:])
        flat = np.concatenate(parts) if n else np.empty(0, dtype=np.uint8)
        if not (n and flat.size):
            return Matches(np.empty(0, dtype=N.MATCH_DTYPE), self._values)
        if narrow:
            return Matches(self._scan_flat(flat, offs, n, 0, algo=algo, sort=sort, device=device, narrow=True), self._values)
        return Matches(self._scan_flat(flat, offs, n, 0, algo=algo, sort=sort, device=device), self._values)


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
