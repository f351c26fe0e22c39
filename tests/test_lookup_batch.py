"""exists_batch / match_batch / longest_prefix_batch / get_batch: the dictionary methods for a whole batch of keys, one
walk from the root per key on the GPU (acb_lookup_device / acb_lookup_host).

The answer is always the drop-in's per-key method (the host trie, which test_api_differential.py checks against the
reference) and, where oracle/_ref is built, the reference extension itself.  Every randomised test has a CPU form on the
numpy restatement of the kernel (tests/emul_lookup.py) and a gpu-marked twin on the real kernel."""
import ctypes

import numpy as np
import pytest

import emul_lookup
import oracle
import pyahocorasick_b200 as pkg
from batch_cases import DT, fake_table, obj, published, skip_if_device
from pyahocorasick_b200 import _native as N
from pyahocorasick_b200 import automaton as am

# (flavour, key type, letters of keys, letters only queries use).  Unicode keys mix latin-1 letters, wider ones and
# non-latin-1 keys with latin-1 prefixes; U+0162 and 0x162 share their low byte with "b" / 0x62, so walks end inside
# a letter.  Bytes-flavour sequences are 2-byte letters, unicode-flavour sequences 4-byte ones.
CASES = {
    "bytes": ("bytes", False, [0x61, 0x62, 0xE9], [0x00, 0x63, 0xFF]),
    "unicode": ("unicode", False, [0x61, 0x62, 0xE9, 0x142, 0x1F600], [0x00, 0x63, 0x162, 0x10FFFF]),
    "seq2": ("bytes", True, [0x61, 0x6162, 0xFF20, 0x62], [0x00, 0x162, 0xFFFF]),
    "seq4": ("unicode", True, [0x61, 0x1F600, 0x10FFFF, 0x62], [0x00, 0x162, 0x7FFFFFFF]),
}
STORES = ["any", "ints", "length"]


def _add(A, store, k, i):
    if store == "length":
        A.add_word(k)
    elif store == "ints":
        A.add_word(k, i * 7 - 3)
    else:
        A.add_word(k, (i, k))


def _pair(case, store, with_ref=True):
    """(drop-in, reference or None) of the same flavour, store and key type"""
    fl, seq = CASES[case][:2]
    out = []
    for mod in (pkg.flavour(fl), oracle.ref_module(fl) if with_ref and oracle.ref_available(fl) else None):
        if mod is None:
            out.append(None)
            continue
        st = {"any": mod.STORE_ANY, "ints": mod.STORE_INTS, "length": mod.STORE_LENGTH}[store]
        out.append(mod.Automaton(st, mod.KEY_SEQUENCE) if seq else mod.Automaton(st))
    return out


def _random_keys(case, rng):
    al = CASES[case][2]
    small = al[:2]                                        # two letters: prefixes collide
    keys = {tuple(int(x) for x in rng.choice(small, size=int(rng.integers(1, 6)))) for _ in range(int(rng.integers(1, 9)))}
    keys |= {tuple(int(x) for x in rng.choice(al, size=int(rng.integers(1, 5)))) for _ in range(int(rng.integers(0, 4)))}
    return [list(k) for k in sorted(keys)]


def _queries(case, keys, rng):
    al, extra = CASES[case][2], CASES[case][3]
    pool = al + extra
    q = [[]]
    for k in keys:
        q.append(k)
        if len(k) > 1:
            q.append(k[:int(rng.integers(1, len(k)))])                                         # proper prefix
        q.append(k + [int(x) for x in rng.choice(pool, size=int(rng.integers(1, 4)))])        # extension
    longest = max(keys, key=len)
    q.append(longest + [int(x) for x in rng.choice(al, size=3)])                                # past the longest key
    q += [[int(x) for x in rng.choice(pool, size=int(rng.integers(1, 7)))] for _ in range(8)]  # letters on no edge too
    q += [[int(rng.choice(extra))]] + [[]]
    order = rng.permutation(len(q))
    return [q[i] for i in order]


def _forms(case, A, queries):
    """every input form the batch methods take (list, (flat, offsets), and uint8[n, stride] for equal lengths)"""
    yield "list", [obj(*CASES[case][:2], x) for x in queries]
    parts = [np.asarray(x, dtype=DT[A._L]).view(np.uint8) for x in queries]
    offs = np.zeros(len(parts) + 1, dtype=np.int64)
    np.cumsum([p.size for p in parts], out=offs[1:])
    yield "flat", (np.concatenate(parts) if parts else np.empty(0, np.uint8), offs)
    if parts and len({p.size for p in parts}) == 1:
        yield "array", np.ascontiguousarray(np.stack(parts))


def _check(A, R, case, queries):
    objs = [obj(*CASES[case][:2], x) for x in queries]
    want = dict(exists=[A.exists(k) for k in objs], match=[A.match(k) for k in objs],
                lp=[A.longest_prefix(k) for k in objs], get=[A.get(k, "dflt") for k in objs])
    if R is not None:
        assert want == dict(exists=[R.exists(k) for k in objs], match=[R.match(k) for k in objs],
                            lp=[R.longest_prefix(k) for k in objs], get=[R.get(k, "dflt") for k in objs]), (case, objs)
    missing = [k for k, e in zip(objs, want["exists"]) if not e]
    for form, x in _forms(case, A, queries):
        e, m, lp = A.exists_batch(x), A.match_batch(x), A.longest_prefix_batch(x)
        assert e.dtype == np.bool_ and m.dtype == np.bool_ and lp.dtype == np.int64
        got = dict(exists=e.tolist(), match=m.tolist(), lp=lp.tolist(), get=A.get_batch(x, "dflt"))
        assert got == want, (case, form, objs)
        if missing:
            with pytest.raises(KeyError) as ei:
                A.get_batch(x)
            assert ei.value.args == (missing[0],), (case, form)
        else:
            assert A.get_batch(x) == want["get"]


def _fuzz(case, store, seed, trials):
    rng = np.random.default_rng(seed)
    for t in range(trials):
        keys = _random_keys(case, rng)
        A, R = _pair(case, store)
        live = {}
        for i, k in enumerate(keys):
            for X in (A, R):
                if X is not None:
                    _add(X, store, obj(*CASES[case][:2], k), i)
            live[tuple(k)] = i
        for X in (A, R):
            if X is not None:
                X.make_automaton()
        _check(A, R, case, _queries(case, keys, rng))
        # the key set changes: remove some (never all: the reference asserts on a lookup in an empty trie), re-add one,
        # or clear and start over; values are replaced in place by add_word of a present key
        op = t % 3
        if op == 0 and len(keys) > 1:
            for k in keys[:len(keys) // 2]:
                for X in (A, R):
                    if X is not None:
                        X.remove_word(obj(*CASES[case][:2], k))
            back = keys[0]
            for X in (A, R):
                if X is not None:
                    _add(X, store, obj(*CASES[case][:2], back), 99)
        elif op == 1:
            for X in (A, R):
                if X is not None:
                    X.clear()
            keys = _random_keys(case, rng)
            for i, k in enumerate(keys):
                for X in (A, R):
                    if X is not None:
                        _add(X, store, obj(*CASES[case][:2], k), 50 + i)
        else:
            for X in (A, R):
                if X is not None:
                    _add(X, store, obj(*CASES[case][:2], keys[-1]), 77)
        for X in (A, R):
            if X is not None:
                X.make_automaton()
        _check(A, R, case, _queries(case, keys, rng))


@pytest.mark.parametrize("store", STORES)
@pytest.mark.parametrize("case", list(CASES))
def test_fuzz_emulated(case, store, monkeypatch):
    emul_lookup.install(monkeypatch)
    _fuzz(case, store, 11, 12)


@pytest.mark.gpu
@pytest.mark.parametrize("store", STORES)
@pytest.mark.parametrize("case", list(CASES))
def test_fuzz_gpu(case, store):
    _fuzz(case, store, 111, 5)


def _root_only(case, store):
    """a built automaton whose keys were all removed before make_automaton: a table of the root alone"""
    A, _ = _pair(case, store, with_ref=False)
    al = CASES[case][2]
    for i, k in enumerate(([al[0]], [al[0], al[1]])):
        _add(A, store, obj(*CASES[case][:2], k), i)
    for k in ([al[0]], [al[0], al[1]]):
        A.remove_word(obj(*CASES[case][:2], k))
    A.make_automaton()
    assert A.kind == pkg.AHOCORASICK and A.flat()["n_states"] == 1
    _check(A, None, case, [[], [al[0]], [al[0], al[1]], [], [CASES[case][3][0]]])
    _check(A, None, case, [[], []])


@pytest.mark.parametrize("case", list(CASES))
def test_empty_keys_and_root_only_table_emulated(case, monkeypatch):
    emul_lookup.install(monkeypatch)
    _root_only(case, "any")


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES))
def test_empty_keys_and_root_only_table_gpu(case):
    _root_only(case, "ints")


# ------------------------------------------------------------------ arguments and states
def test_unbuilt_automata_raise_what_find_all_batch_raises(monkeypatch):
    emul_lookup.install(monkeypatch)
    mod = pkg.flavour("bytes")
    A = mod.Automaton()
    for step in ("empty", "trie"):
        with pytest.raises(AttributeError) as want:
            A.find_all_batch([b"a"])
        for name in ("exists_batch", "match_batch", "longest_prefix_batch", "get_batch"):
            with pytest.raises(AttributeError) as got:
                getattr(A, name)([b"a"])
            assert str(got.value) == str(want.value)
        A.add_word(b"ab", 1)
    A.make_automaton()
    assert A.exists_batch([b"ab", b"a"]).tolist() == [True, False]
    A.add_word(b"ab", 2)                                  # the key set is a trie again until make_automaton
    assert A.exists(b"ab") and A.get(b"ab") == 2          # the per-key methods keep working on it
    with pytest.raises(AttributeError):
        A.exists_batch([b"ab"])
    A.make_automaton()
    assert A.get_batch([b"ab"]) == [2]                    # values replaced in place are read at call time


def _error(fn):
    try:
        fn()
    except (TypeError, ValueError) as e:
        return type(e), str(e)
    return None


@pytest.mark.parametrize("fl, seq, good, bad", [
    ("bytes", False, b"ab", ["ab", 3]),
    ("unicode", False, "ab", [b"ab", 3]),
    ("bytes", True, (97, 98), [("x",), (-1,), b"ab"]),
    ("unicode", True, (97, 98), [(1.5,), (2 ** 32,), "ab"]),
])
def test_wrong_keys_raise_the_per_key_errors(fl, seq, good, bad, monkeypatch):
    emul_lookup.install(monkeypatch)
    mod = pkg.flavour(fl)
    A = mod.Automaton(mod.STORE_ANY, mod.KEY_SEQUENCE) if seq else mod.Automaton()
    A.add_word(good, 1)
    A.make_automaton()
    for i in range(len(bad)):
        batch = [good] + bad[i:]                          # the first offending key decides
        want = _error(lambda: A.exists(bad[i]))
        assert want is not None
        for name in ("exists_batch", "match_batch", "longest_prefix_batch", "get_batch"):
            assert _error(lambda: getattr(A, name)(batch)) == want, (name, batch)
        for name in ("exists", "match", "longest_prefix", "get"):
            assert _error(lambda: getattr(A, name)(bad[i])) == want


def test_get_batch_keyerror_names_the_first_missing_key_in_every_form(monkeypatch):
    emul_lookup.install(monkeypatch)
    for fl, keys, miss in (("bytes", [b"abc", b"abd"], b"abx"), ("unicode", ["abc", "abł"], "aŢx")):
        A = pkg.flavour(fl).Automaton()
        for k in keys:
            A.add_word(k, k.upper())
        A.make_automaton()
        batch = [keys[0], miss, "zzz" if fl == "unicode" else b"zzz"]
        with pytest.raises(KeyError) as e:
            A.get_batch(batch)
        assert e.value.args == (miss,)
        with pytest.raises(KeyError) as e:
            A.get_batch(iter(batch))
        assert e.value.args == (miss,)
        with pytest.raises(KeyError) as e:
            A.get(miss)
        assert e.value.args == (miss,)
        assert A.get_batch(batch, None) == [keys[0].upper(), None, None]
        raw = np.stack([np.frombuffer(A._raw_key(k)[0], dtype=np.uint8) for k in batch])
        with pytest.raises(KeyError) as e:
            A.get_batch(raw)
        assert e.value.args == (miss,)


def test_str_lists_take_one_join_with_the_bytes_of_the_per_item_path():
    A = pkg.flavour("unicode").Automaton()
    lists = [["ab", "", "ł\U0001F600", "\ud800", "\udc00", "x" * 40, "\xe9"], ["\U0010FFFF"], [""]]
    for keys in lists:
        fast = A._batch_input(keys, narrow_ok=False)
        per_item = [A._letters(k) for k in keys]
        flat = np.concatenate([p.view(np.uint8) for p in per_item])
        offs = np.concatenate([[0], np.cumsum([p.nbytes for p in per_item])]).astype(np.int64)
        assert fast[0] == "host" and fast[3] == len(keys) and fast[4] == 0 and fast[5] is False
        assert fast[1].tobytes() == flat.tobytes() and fast[2].tolist() == offs.tolist()
        mixed = A._batch_input(keys + [np.str_("q")], narrow_ok=False)       # a str subclass: the per-item path
        assert mixed[1].tobytes() == flat.tobytes() + "q".encode("utf-32-le")
        assert mixed[2].tolist() == offs.tolist() + [offs[-1] + 4]
    assert A._batch_input(["ab"], narrow_ok=True)[5] is True                               # scans keep the latin-1 path


def test_lookup_host_fails_loudly_without_a_device():
    skip_if_device()
    L = N.lib()
    fake = fake_table()                                   # device 0, and no device to select
    keys = np.frombuffer(b"abcd", dtype=np.uint8)
    offs = np.array([0, 2, 4], dtype=np.int64)
    kid, pre = np.empty(2, np.int32), np.empty(2, np.int32)
    assert L.acb_lookup_host(ctypes.addressof(fake), N.ptr(keys), 4, N.ptr(offs), 2, 0, N.ptr(kid), N.ptr(pre)) == N.ACB_ECUDA
    assert N.last_error()
    assert L.acb_lookup_host(None, N.ptr(keys), 4, N.ptr(offs), 2, 0, N.ptr(kid), N.ptr(pre)) == N.ACB_EINVAL
    assert L.acb_lookup_device(None, N.ptr(keys), 4, None, 2, 2, N.ptr(kid), N.ptr(pre), None) == N.ACB_EINVAL
    A = pkg.flavour("bytes").Automaton()
    A.add_word(b"ab", 1)
    A.make_automaton()
    with pytest.raises(N.NativeError):                    # no CPU fallback behind the Python methods either
        A.exists_batch([b"ab"])


# ------------------------------------------------------------------ GPU only
def _per_key(A, objs):
    return ([A.exists(k) for k in objs], [A.match(k) for k in objs], [A.longest_prefix(k) for k in objs],
            [A.get(k, None) for k in objs])


def _batch(A, x):
    return (A.exists_batch(x).tolist(), A.match_batch(x).tolist(), A.longest_prefix_batch(x).tolist(), A.get_batch(x, None))


@pytest.mark.gpu
def test_all_256_byte_values_on_edges():
    A = pkg.flavour("bytes").Automaton(pkg.STORE_INTS)
    for b in range(256):
        A.add_word(bytes([b, 0x71]), b)
    A.add_word(b"\x00\x00\x00", 1000)
    A.add_word(b"\xff\x00", 1001)
    A.make_automaton()
    assert A.flat()["n_classes"] == 256                   # class 0 is the byte 0x00, a real edge
    q = [bytes([b]) for b in range(256)] + [bytes([b, 0x71]) for b in range(256)] + [bytes([b, 0x70]) for b in range(256)]
    q += [b"\x00", b"\x00\x00", b"\x00\x00\x00", b"\x00\x00\x00\x00", b"\xff\x00", b"\xff\x00\x00", b""]
    assert _batch(A, q) == _per_key(A, q)
    assert A.longest_prefix_batch([b"\x00\x00\x00\x00"]).tolist() == [3]


@pytest.mark.gpu
def test_goto_table_past_2_31_entries():
    rng = np.random.default_rng(5)
    raw = rng.integers(0, 256, size=(800_000, 14), dtype=np.uint8)
    keys = [bytes(r) for r in raw]
    A = pkg.flavour("bytes").Automaton(pkg.STORE_INTS)
    for i, k in enumerate(keys):
        A.add_word(k, i)
    A.make_automaton()
    fv = N.FlatView()
    N.check(A._lib.acb_trie_flat_view(A._trie, ctypes.byref(fv)))
    assert fv.n_classes * fv.n_states > 2 ** 31, (fv.n_classes, fv.n_states)
    pick = rng.permutation(len(keys))[:20_000]
    q = [keys[i] for i in pick[:8000]]
    q += [keys[i][:int(rng.integers(1, 14))] for i in pick[8000:14000]]
    q += [keys[i][:13] + bytes([(keys[i][13] + 1) % 256]) for i in pick[14000:17000]]
    q += [keys[i] + b"\xff" for i in pick[17000:]]
    assert _batch(A, q) == _per_key(A, q)
    got = A.get_batch([keys[i] for i in pick])
    assert got == pick.tolist()


@pytest.mark.gpu
def test_walks_that_end_inside_a_letter():
    """letters of 1, 2 and 4 bytes whose low bytes are those of the keys: a letter walked only in part does not count"""
    B = pkg.flavour("bytes").Automaton()
    for k in (b"ab", b"abc"):
        B.add_word(k, k)
    B.make_automaton()
    q = [b"ab", b"abd", b"a", b"abcd", b"b"]
    assert _batch(B, q) == _per_key(B, q)
    S = pkg.flavour("bytes").Automaton(pkg.STORE_ANY, pkg.KEY_SEQUENCE)
    for k in ((0x61, 0x62), (0x61, 0x62, 0x63)):
        S.add_word(k, k)
    S.make_automaton()
    q = [(0x61, 0x162), (0x61, 0x62, 0x163), (0x61, 0x62, 0x6300), (0x161,), (0x61, 0x62)]
    assert _batch(S, q) == _per_key(S, q)
    assert S.longest_prefix_batch(q).tolist() == [1, 2, 2, 0, 2]
    U = pkg.flavour("unicode").Automaton()
    for k in ("ab", "abc"):
        U.add_word(k, k)
    U.make_automaton()
    q = ["aŢ", "ab\U00010063", "abţ", "š", "abc", "ab\x63\x00"]
    assert _batch(U, q) == _per_key(U, q)
    assert U.longest_prefix_batch(q).tolist() == [1, 2, 2, 0, 3, 3]
    assert U.match_batch(q).tolist() == [False, False, False, False, True, False]


@pytest.mark.gpu
def test_fixed_stride_kmers():
    rng = np.random.default_rng(9)
    A = pkg.flavour("bytes").Automaton(pkg.STORE_INTS)
    al = np.frombuffer(b"ACGT", dtype=np.uint8)
    kmers = rng.choice(al, size=(5000, 8))
    for i, k in enumerate(kmers):
        A.add_word(k.tobytes(), i)
    A.make_automaton()
    q = np.ascontiguousarray(np.concatenate([kmers[:3000], rng.choice(al, size=(3000, 8))]))
    objs = [r.tobytes() for r in q]
    assert _batch(A, q) == _per_key(A, objs)
    assert _batch(A, np.zeros((4, 0), dtype=np.uint8)) == _per_key(A, [b""] * 4)


@pytest.mark.gpu
@pytest.mark.parametrize("fl", ["bytes", "unicode"])
def test_cuda_tensors_on_a_side_stream(fl):
    import torch
    rng = np.random.default_rng(4)
    A = pkg.flavour(fl).Automaton(pkg.STORE_INTS)
    L = A._L
    letters = [0x61, 0x62, 0x163] if fl == "unicode" else [0x61, 0x62]
    keys = {tuple(int(x) for x in rng.choice(letters[:2], size=int(rng.integers(1, 4)))) for _ in range(12)}
    for i, k in enumerate(sorted(keys)):
        A.add_word(obj(fl, False, list(k)), i)
    A.make_automaton()
    rows = rng.choice(letters, size=(2001, 7 if L == 1 else 2)).astype(DT[L])
    host = np.ascontiguousarray(rows.view(np.uint8).reshape(2001, -1))
    d = torch.from_numpy(host).cuda()
    views = {"whole": (d, host), "misaligned": (d[1:], host[1:])}
    assert d[1:].data_ptr() % 16 != 0 or L != 1
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    for name, (t, h) in views.items():
        with torch.cuda.stream(side):
            e, m, lp = A.exists_batch(t), A.match_batch(t), A.longest_prefix_batch(t)
            got_get = A.get_batch(t, None)
        assert e.is_cuda and m.is_cuda and lp.is_cuda and e.dtype == torch.bool and lp.dtype == torch.int64
        side.synchronize()
        objs = [_row_obj(A, r) for r in h]
        assert (e.cpu().tolist(), m.cpu().tolist(), lp.cpu().tolist(), got_get) == _per_key(A, objs), name


def _row_obj(A, r):
    raw = r.tobytes()
    return raw.decode("utf-32-le") if A._L == 4 else raw


@pytest.mark.gpu
def test_queries_past_2_31_bytes():
    """int64 offsets: 2^27 + 2 queries, the last ones starting past 2^31 bytes; answers checked by construction and on
    a sample with the per-key methods"""
    A = pkg.flavour("bytes").Automaton(pkg.STORE_INTS)
    words = [bytes([65 + i]) * 16 for i in range(7)]
    for i, w in enumerate(words):
        A.add_word(w, i)
    A.add_word(b"Z" * 16 + b"tail", 7)
    A.make_automaton()
    block = np.frombuffer(b"".join(words) + b"A" * 15 + b"B", dtype=np.uint8)       # 8 queries of 16 bytes
    reps = (1 << 27) // 8
    tail = np.frombuffer(b"Z" * 16 + b"tail" + b"Z" * 16 + b"ta", dtype=np.uint8)
    flat = np.concatenate([np.tile(block, reps), tail])
    n = reps * 8
    offs = np.concatenate([np.arange(n + 1, dtype=np.int64) * 16, [n * 16 + 20, n * 16 + 38]]).astype(np.int64)
    assert offs[-2] > 2 ** 31 and offs[-1] == flat.size
    kid = A.get_batch((flat, offs), -1)
    want_block = list(range(7)) + [-1]
    assert kid[:8] == want_block and kid[n - 8:n] == want_block and kid[n:] == [7, -1]
    kid = np.asarray(kid)
    assert (kid[:n].reshape(-1, 8) == np.array(want_block)).all()
    lp = A.longest_prefix_batch((flat, offs))
    assert lp[7] == 15 and lp[n] == 20 and lp[n + 1] == 18
    rng = np.random.default_rng(2)
    for i in rng.integers(0, n + 2, size=500).tolist() + [n, n + 1]:
        k = flat[offs[i]:offs[i + 1]].tobytes()
        assert (bool(kid[i] >= 0), int(lp[i])) == (A.exists(k), A.longest_prefix(k)), i


@pytest.mark.gpu
def test_published_lookup_shape_in_full():
    """1 M words of 3..32 characters over [a-zA-Z0-9], each its own value; 1 M present and 1 M absent lookups"""
    pw = published(1_000_000, n_missing=1_000_000)
    words = [w.encode() for w in pw.words]
    missing = [w.encode() for w in pw.missing]
    del pw
    A = pkg.flavour("bytes").Automaton()
    for w in words:
        A.add_word(w, w)
    A.make_automaton()
    q = words + missing
    assert A.get_batch(q, None) == [A.get(w, None) for w in q]
    assert A.get_batch(words) == words
    assert A.exists_batch(q).tolist() == [True] * len(words) + [False] * len(missing)


@pytest.mark.gpu
def test_unicode_answers_come_from_the_full_table_after_a_latin1_scan():
    A = pkg.flavour("unicode").Automaton()
    for k in ("xy", "abłd", "\xe9t\xe9"):
        A.add_word(k, k)
    A.make_automaton()
    m = A.find_all_batch(["..xy..", "\xe9t\xe9"])           # latin-1 haystacks: builds and uploads the latin-1 table
    assert len(m) == 2 and A._narrow_table is not None
    q = ["ab", "abł", "abłd", "abłdd", "xy", "x", "\xe9t", "\xe9t\xe9", "q", ""]
    assert _batch(A, q) == _per_key(A, q)
    assert A.match_batch(["ab"]).tolist() == [True] and A.longest_prefix_batch(["abł"]).tolist() == [3]


@pytest.mark.gpu
def test_c_entries_check_their_arguments():
    A = pkg.flavour("unicode").Automaton()
    A.add_word("ab", 1)
    A.make_automaton()
    tb = A._ensure_table(0)
    L = N.lib()
    keys = np.frombuffer("abab".encode("utf-32-le"), dtype=np.uint8)
    kid, pre = np.empty(2, np.int32), np.empty(2, np.int32)
    for offs in ([0, 8, 12], [4, 8, 16], [0, 12, 8], [0, 6, 16]):               # wrong end, start, order, letter cut
        o = np.array(offs, dtype=np.int64)
        assert L.acb_lookup_host(tb, N.ptr(keys), 16, N.ptr(o), 2, 0, N.ptr(kid), N.ptr(pre)) == N.ACB_EINVAL, offs
    assert L.acb_lookup_host(tb, N.ptr(keys), 16, None, 2, 6, N.ptr(kid), N.ptr(pre)) == N.ACB_EINVAL
    assert L.acb_lookup_host(tb, N.ptr(keys), 16, None, 3, 8, N.ptr(kid), N.ptr(pre)) == N.ACB_EINVAL
    assert L.acb_lookup_host(tb, N.ptr(keys), 16, None, 2, 8, N.ptr(kid), N.ptr(pre)) == N.ACB_OK
    assert kid.tolist() == [0, 0] and pre.tolist() == [2, 2]
    o = np.array([0, 4, 16], dtype=np.int64)
    assert L.acb_lookup_host(tb, N.ptr(keys), 16, N.ptr(o), 2, 0, N.ptr(kid), N.ptr(pre)) == N.ACB_OK
    assert kid.tolist() == [-1, -1] and pre.tolist() == [1, 0]
