"""Cases, input forms, references and C-entry checks shared by the batch-feature tests (leftmost-longest, replacement,
whole words, white space, lookups, selects, stream batches).  Not a test module: tests/conftest.py puts tests/ on the
path, and the test modules import from here, never from each other."""
import collections
import ctypes
import random
import string

import numpy as np
import pytest

import oracle
import pyahocorasick_b200 as pkg
from pyahocorasick_b200 import _native as N

DT = {1: np.uint8, 2: "<u2", 4: "<u4"}            # letter width -> dtype of one letter

# (flavour, key type, text alphabet): latin-1, wide and mixed unicode; bytes-flavour sequences are 2-byte letters,
# unicode-flavour sequences 4-byte ones
CASES = {
    "bytes": ("bytes", False, [0x61, 0x62, 0xE9]),
    "latin1": ("unicode", False, [0x61, 0x62, 0xE9]),
    "wide": ("unicode", False, [0x61, 0x142, 0x1F600]),
    "mixed": ("unicode", False, [0x61, 0x62, 0x1F600]),
    "seq2": ("bytes", True, [0x61, 0x6162, 0xFF20]),
    "seq4": ("unicode", True, [0x61, 0x1F600, 0x10FFFF]),
}

NESTED = [[0x61] * k for k in range(1, 17)]                               # a ... a^16


def obj(fl, seq, letters):
    """letters as the drop-in takes them: a tuple for key sequences, else bytes or str"""
    if seq:
        return tuple(letters)
    return bytes(letters) if fl == "bytes" else "".join(map(chr, letters))


def automaton(fl, seq, keys, mp=None, env=None, tagmap=False):
    """the drop-in (STORE_INTS, value = index) and the C oracle over the same keys, given as letters; env forces
    ACB_FILTER (and tagmap ACB_FORCE_TAGMAP) through the monkeypatch mp, around make_automaton only"""
    mod = pkg.flavour(fl)
    A = mod.Automaton(mod.STORE_INTS, mod.KEY_SEQUENCE) if seq else mod.Automaton(mod.STORE_INTS)
    O = oracle.OracleAutomaton()
    for i, k in enumerate(keys):
        A.add_word(obj(fl, seq, k), i)
        O.add_word(obj(fl, seq, k), i)
    if env is None:
        A.make_automaton()
    else:
        with mp.context() as m:
            m.setenv("ACB_FILTER", env)
            if tagmap:
                m.setenv("ACB_FORCE_TAGMAP", "1")
            A.make_automaton()
    O.make_automaton()
    return A, O


def layout(seqs, width):
    """letter sequences as one batch: (flat uint8, int64 byte offsets)"""
    dt = DT[width]
    parts = [np.asarray(s, dtype=dt).view(np.uint8) for s in seqs]
    offs = np.zeros(len(parts) + 1, dtype=np.int64)
    np.cumsum([p.size for p in parts], out=offs[1:])
    return (np.concatenate(parts) if parts else np.empty(0, np.uint8)), offs


def split(out, offs, width):
    """a (flat, byte offsets) batch back into per-haystack letter lists"""
    dt = DT[width]
    return [np.asarray(out[offs[i]:offs[i + 1]]).view(dt).tolist() for i in range(len(offs) - 1)]


def forms(objs, hays, L, list_only):
    """the input forms of find_all_batch for one batch: the list of objects and, unless list_only, (flat, offsets) and,
    when every haystack has the same non-zero length, uint8[n, stride]"""
    yield "list", objs
    if list_only:
        return
    flat, offs = layout(hays, L)
    yield "flat", (flat, offs)
    width = max(len(h) for h in hays)
    if width and all(len(h) == width for h in hays):
        yield "array", flat.reshape(len(hays), -1)


def oracle_full(O, hays, case="bytes"):
    """the C oracle's full list [(hay, end, value)]; bytes-flavour text letters as the reference widens them"""
    fl, seq, _ = CASES[case]
    letters = np.array([x for h in hays for x in h], dtype=np.uint32)
    if fl == "bytes" and not seq:
        letters = oracle._letters(letters.astype(np.uint8).tobytes())
    offs = np.zeros(len(hays) + 1, dtype=np.int64)
    np.cumsum([len(h) for h in hays], out=offs[1:])
    return O.scan_batch_letters(letters, offs)


def rows(m):
    """a Matches as int64 rows (hay_id, end_index, key_id)"""
    return np.stack([m.hay_id.astype(np.int64), m.end_index.astype(np.int64), m.key_id.astype(np.int64)], axis=1)


def triples(m):
    """a Matches as [(hay_id, end_index, key_id)]"""
    return list(zip(m.hay_id.tolist(), m.end_index.tolist(), m.key_id.tolist()))


def got_values(m):
    """a Matches as [(hay_id, end_index, value)]"""
    return list(zip(m.hay_id.tolist(), m.end_index.tolist(), m.values()))


def key_len(A):
    return np.asarray(A.flat()["key_len"], dtype=np.int64)


def table_and_batch(A, hays):
    """the device-0 table and a bytes batch as (flat, offsets) for the C entries"""
    flat = np.frombuffer(b"".join(hays), dtype=np.uint8).copy()
    offs = np.zeros(len(hays) + 1, dtype=np.int64)
    np.cumsum([len(h) for h in hays], out=offs[1:])
    return A._ensure_table(0), flat, offs


def np_greedy(full: np.ndarray, key_len: np.ndarray) -> np.ndarray:
    """the leftmost-longest definition over a full record array (hay_id, end_index, key_id), vectorised but for the walk
    itself"""
    if len(full) == 0:
        return np.empty((0, 3), dtype=np.int64)
    hay, end, key = (full[f].astype(np.int64) for f in ("hay_id", "end_index", "key_id"))
    ln = key_len[key]
    start = end - ln + 1
    o = np.lexsort((-ln, start, hay))
    hay, start, ln, end, key = hay[o], start[o], ln[o], end[o], key[o]
    first = np.ones(len(o), dtype=bool)
    first[1:] = (hay[1:] != hay[:-1]) | (start[1:] != start[:-1])
    hay, start, ln, end, key = hay[first], start[first], ln[first], end[first], key[first]
    big = np.int64(1) << 32                                 # start + len < 2^32: one sortable number per (hay, start)
    flat = hay * big + start
    nxt = np.searchsorted(flat, flat + ln)
    nxt_ok = nxt < len(flat)
    nxt_ok[nxt_ok] = hay[nxt[nxt_ok]] == hay[nxt_ok]
    heads = np.nonzero(np.r_[True, hay[1:] != hay[:-1]])[0].tolist()
    nx = np.where(nxt_ok, nxt, -1).tolist()
    chosen = []
    for i in heads:
        while i >= 0:
            chosen.append(i)
            i = nx[i]
    chosen = np.array(sorted(chosen), dtype=np.int64)
    return np.stack([hay[chosen], end[chosen], key[chosen]], axis=1)


# ------------------------------------------------------------------ the reference's published benchmark shape
PUBLISHED_CHARS = string.ascii_letters + string.digits


Published = collections.namedtuple("Published", "words text missing")


def _published_word(rng):
    return "".join(rng.choice(PUBLISHED_CHARS) for _ in range(rng.randint(3, 32)))


def published(n, text_length=0, n_missing=0):
    """the reference's published benchmark shape (etc/benchmarks/benchmark.py), drawn in one pass of random.Random(0):
    n distinct words of 3..32 characters over [A-Za-z0-9] as str, in generation order (not a set's order, which changes
    with PYTHONHASHSEED and with it the key ids); then the haystack of text_length characters, drawn right after the
    words as tools/published_benchmark.py draws it; then n_missing distinct words of the same shape that are not keys.
    Nothing is cached: the caller decides how long the million strings live."""
    rng = random.Random(0)
    seen = {}
    while len(seen) < n:
        seen.setdefault(_published_word(rng))
    text = "".join(rng.choice(PUBLISHED_CHARS) for _ in range(text_length))
    missing = {}
    while len(missing) < n_missing:
        w = _published_word(rng)
        if w not in seen:
            missing.setdefault(w)
    return Published(list(seen), text, list(missing))


def published_words(n):
    """published(n).words"""
    return published(n).words


# ------------------------------------------------------------------ random and structured cases of more than one file
def leftmost_random_case(case, rng):
    _, _, al = CASES[case]
    keys = sorted({tuple(int(x) for x in rng.choice(al[:2] if rng.integers(0, 2) else al, size=int(rng.integers(1, 7))))
                   for _ in range(int(rng.integers(1, 9)))})
    hays = []
    for _ in range(int(rng.integers(1, 10))):
        r = int(rng.integers(0, 6))
        if r == 0:
            hays.append([])
        elif r == 1:
            hays.append([0x63] * int(rng.integers(1, 5)) if case != "seq2" else [0x7A])          # no match
        else:
            hays.append([int(x) for x in rng.choice(al, size=int(rng.integers(1, 50)))])
    if case == "mixed" and all(max(h, default=0) < 256 for h in hays):
        hays.append([0x1F600, 0x61, 0x62])
    return keys, hays


def leftmost_structured_cases():
    """nested keys, prefixes and suffixes of others, adjacent and abutting matches, empty haystacks, no match"""
    a, b, c = 0x61, 0x62, 0x63
    yield NESTED, [[a] * 40, [a] * 16 + [b] + [a] * 17, [], [b, b], [a, b] * 9, [a]]
    yield [[a, b], [a, b, c], [b, c], [c], [b, c, a, b]], [[a, b, c, a, b, c], [a, b, a, b, a, b], [c, c, c], [], [b, c, a, b, c]]
    yield [[a, b, c, 0x64, 0x65], [b, c, 0x64, 0x78], [c, 0x64]], [[a, b, c, 0x64, 0x79]]      # the documented example
    yield [[a, b], [b, a]], [[a, b, a, b, a], [b, a, b], [a], [b]]


def replace_reps(case, keys, rng):
    """a replacement per key: empty, shorter, equal (the key itself), longer, or text that holds other keys"""
    al = CASES[case][2]
    out = []
    for k in keys:
        r = int(rng.integers(0, 5))
        if r == 0:
            out.append([])
        elif r == 1:
            out.append(list(k[: max(len(k) - 1, 0)]))
        elif r == 2:
            out.append(list(k))
        elif r == 3:
            out.append([int(x) for x in rng.choice(al, size=len(k) + int(rng.integers(1, 5)))])
        else:
            out.append(list(keys[int(rng.integers(0, len(keys)))]) * 2)
    return out


# ------------------------------------------------------------------ the C entries
def fake_table(L=0):
    """a zeroed stand-in for acb_table (device 0) with the letter width set: acb_table starts with int device, int
    sm_count, int32 S, K, L"""
    fake = ctypes.create_string_buffer(1 << 16)
    ctypes.c_int32.from_buffer(fake, 16).value = L
    return fake


def skip_if_device():
    """for the tests of the ACB_ECUDA an entry returns when no device can be used"""
    import torch
    if torch.cuda.is_available():
        pytest.skip("a device is present")


def check_host_capacities(call, want):
    """a host entry that returns records, at capacities 0, 1, n-1 and n: the exact count every time, ACB_EOVERFLOW
    below n, the records (int64 rows) at n.  call(out, cap, found) passes its arguments on to the entry"""
    n = len(want)
    found = ctypes.c_int64(0)
    for cap in (0, 1, n - 1, n):
        out = np.zeros(max(cap, 1), dtype=N.MATCH_DTYPE)
        rc = call(N.ptr(out), cap, ctypes.byref(found))
        assert found.value == n
        assert rc == (N.ACB_OK if cap >= n else N.ACB_EOVERFLOW)
        if cap >= n:
            assert np.array_equal(np.stack([out["hay_id"], out["end_index"], out["key_id"]], axis=1)[:n].astype(np.int64), want)


def check_device_capacities(call, want, d_records):
    """a device entry that adds to a record buffer, at capacities 0, 1, n-1 and n: rows filled with -7 and a count preset
    to 5, so the count is added to, the records land after the first 5 slots, slots before *d_count and rows at or past
    the capacity stay untouched, and d_records is not changed.  call(out, cap, count, stream) passes its arguments on"""
    import torch
    n = len(want)
    before = d_records.cpu().numpy()
    for cap in (0, 1, n - 1, n):
        out = torch.full((cap + 4, 3), -7, dtype=torch.int32, device="cuda")
        cnt = torch.tensor([5], dtype=torch.int64, device="cuda")
        assert call(out.data_ptr(), cap, cnt.data_ptr(), torch.cuda.current_stream().cuda_stream) == N.ACB_OK
        assert int(cnt.item()) == 5 + n
        o = out.cpu().numpy()
        assert (o[cap:] == -7).all()
        if cap > 5:
            assert np.array_equal(o[5:cap].astype(np.int64), want[:cap - 5])
        assert (o[:min(cap, 5)] == -7).all()
    assert np.array_equal(before, d_records.cpu().numpy())
