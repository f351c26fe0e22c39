"""select_batch / keys_batch / values_batch / items_batch: keys / values / items (prefix, wildcard, how) for a whole batch
of patterns in one GPU call (acb_select_device / acb_select_host).

The answer is always the drop-in's per-key method (the host trie's enumeration, which test_api_differential.py checks
against the reference) and, where oracle/_ref is built, the reference extension itself.  Every randomised test has a CPU
form on the Python restatement of the kernel (tests/emul_select.py) and a gpu-marked twin on the real kernel."""
import ctypes
import os
import pickle
import string

import numpy as np
import pytest

import emul_select
import oracle
import pyahocorasick_b200 as pkg
from batch_cases import DT, fake_table, obj, published_words, skip_if_device
from pyahocorasick_b200 import _native as N

EXACT, AT_MOST, AT_LEAST = pkg.MATCH_EXACT_LENGTH, pkg.MATCH_AT_MOST_PREFIX, pkg.MATCH_AT_LEAST_PREFIX
HOWS = [EXACT, AT_MOST, AT_LEAST]

# (flavour, key type, letters of keys, letters only patterns use).  U+0162 and 0x162 share their low byte with "b" /
# 0x62, so plain letters of a pattern can end a walk inside a letter.
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
    keys = {tuple(int(x) for x in rng.choice(small, size=int(rng.integers(1, 6)))) for _ in range(int(rng.integers(1, 12)))}
    keys |= {tuple(int(x) for x in rng.choice(al, size=int(rng.integers(1, 5)))) for _ in range(int(rng.integers(0, 5)))}
    keys = [list(k) for k in keys]
    rng.shuffle(keys)                                     # insertion order decides the key order
    return keys


def _patterns(case, keys, rng, w):
    """prefixes, keys, extensions, letters on no edge, all-wildcard patterns, the empty pattern, patterns past the
    longest key; with a wildcard w, random letters of each replaced by it"""
    al, extra = CASES[case][2], CASES[case][3]
    pool = al + extra
    q = [[]]
    for k in keys:
        q.append(k)
        if len(k) > 1:
            q.append(k[:int(rng.integers(1, len(k)))])
        q.append(k + [int(x) for x in rng.choice(pool, size=int(rng.integers(1, 3)))])
    longest = max(len(k) for k in keys)
    q += [[int(x) for x in rng.choice(pool, size=int(rng.integers(1, 6)))] for _ in range(5)]
    q.append([int(x) for x in rng.choice(al, size=longest + 2)])
    if w is not None:
        q = [[w if rng.random() < 0.4 else x for x in p] for p in q]
        q += [[w] * i for i in range(longest + 3)]
    order = rng.permutation(len(q))
    return [q[i] for i in order]


def _forms(case, A, patterns):
    """every input form the batch methods take (list, (flat, offsets), and uint8[n, stride] for equal lengths)"""
    yield "list", [obj(*CASES[case][:2], x) for x in patterns]
    parts = [np.asarray(x, dtype=DT[A._L]).view(np.uint8) for x in patterns]
    offs = np.zeros(len(parts) + 1, dtype=np.int64)
    np.cumsum([p.size for p in parts], out=offs[1:])
    yield "flat", (np.concatenate(parts) if parts else np.empty(0, np.uint8), offs)
    same = [p for p in parts if p.size == parts[0].size] if parts else []
    if len(same) > 1:
        yield "array", np.ascontiguousarray(np.stack(same))


def _rows(case, A, x):
    """the patterns of an input form as objects"""
    if isinstance(x, list):
        return x
    if isinstance(x, tuple):
        flat, offs = x
        raw = [flat[offs[i]:offs[i + 1]].tobytes() for i in range(len(offs) - 1)]
    else:
        raw = [r.tobytes() for r in x]
    return [obj(*CASES[case][:2], np.frombuffer(r, dtype=DT[A._L]).tolist()) for r in raw]


def _check(A, R, case, patterns, w, how):
    wobj = None if w is None else obj(*CASES[case][:2], [w])
    for form, x in _forms(case, A, patterns):
        objs = _rows(case, A, x)
        want_k = [list(A.keys(p, wobj, how)) for p in objs]
        want_v = [list(A.values(p, wobj, how)) for p in objs]
        want_i = [list(A.items(p, wobj, how)) for p in objs]
        assert A.keys_batch(x, wobj, how) == want_k, (case, form, w, how)
        assert A.values_batch(x, wobj, how) == want_v, (case, form, w, how)
        assert A.items_batch(x, wobj, how) == want_i, (case, form, w, how)
        offs, kid = A.select_batch(x, wobj, how)
        assert offs.dtype == np.int64 and kid.dtype == np.int32 and len(offs) == len(objs) + 1
        if R is not None and form == "list" and not CASES[case][1]:
            # the reference takes no None wildcard (it raises "string expected"); a prefix alone is its prefix query,
            # which is what the drop-in answers for (p, None, how) whatever how is.  Its keys() reads the pattern as a
            # string also for KEY_SEQUENCE automata (pymod_get_string, src/Automaton.c:747), so tuple patterns are
            # compared with the drop-in's per-key methods only
            rargs = () if wobj is None else (wobj, how)
            assert [list(R.values(p, *rargs)) for p in objs] == want_v, (case, w, how)
            if CASES[case][0] == "unicode":           # the bytes reference mangles the keys it yields (DESIGN §8)
                assert [list(R.keys(p, *rargs)) for p in objs] == want_k, (case, w, how)
                assert [list(R.items(p, *rargs)) for p in objs] == want_i, (case, w, how)


def _check_all(A, R, case, keys, rng):
    al, extra = CASES[case][2], CASES[case][3]
    for w in (None, al[0], extra[0]):                     # none, a letter of the keys, a letter of no key
        pats = _patterns(case, keys, rng, w)
        for how in HOWS:
            _check(A, R, case, pats, w, how)


def _fuzz(case, store, seed, trials):
    rng = np.random.default_rng(seed)
    for t in range(trials):
        keys = _random_keys(case, rng)
        A, R = _pair(case, store)
        for i, k in enumerate(keys):
            for X in (A, R):
                if X is not None:
                    _add(X, store, obj(*CASES[case][:2], k), i)
        for X in (A, R):
            if X is not None:
                X.make_automaton()
        _check_all(A, R, case, keys, rng)
        # remove some keys and add them back: a re-linked node becomes its parent's youngest child
        if len(keys) > 1:
            gone = keys[:len(keys) // 2]
            for k in gone:
                for X in (A, R):
                    if X is not None:
                        X.remove_word(obj(*CASES[case][:2], k))
            for k in gone[::-1][:2]:
                for X in (A, R):
                    if X is not None:
                        _add(X, store, obj(*CASES[case][:2], k), 90)
            keys = keys[len(keys) // 2:] + gone[::-1][:2]
        for X in (A, R):
            if X is not None:
                X.make_automaton()
        _check_all(A, R, case, keys, rng)


@pytest.mark.parametrize("store", STORES)
@pytest.mark.parametrize("case", list(CASES))
def test_fuzz_emulated(case, store, monkeypatch):
    emul_select.install(monkeypatch)
    _fuzz(case, store, 21, 3)


@pytest.mark.gpu
@pytest.mark.parametrize("store", STORES)
@pytest.mark.parametrize("case", list(CASES))
def test_fuzz_gpu(case, store):
    _fuzz(case, store, 121, 3)


@pytest.mark.parametrize("case", list(CASES))
def test_key_ranges_restate_the_key_order(case):
    """order is acb_trie_key_order; every letter state's run holds exactly the keys at or under it; children are youngest
    first, by ascending lo, and their runs tile the parent's after its own key"""
    rng = np.random.default_rng(3)
    A, _ = _pair(case, "ints", with_ref=False)
    keys = _random_keys(case, rng) + _random_keys(case, rng)
    for i, k in enumerate(keys):
        _add(A, "ints", obj(*CASES[case][:2], k), i)
    for k in keys[::3]:
        A.remove_word(obj(*CASES[case][:2], k))
    for k in keys[::6]:
        _add(A, "ints", obj(*CASES[case][:2], k), 5)
    A.make_automaton()
    f, kr = A.flat(), A.key_ranges()
    want = [A._key_ids[k] for k in A.keys()]
    assert kr["order"].tolist() == want
    lo, cnt, cp, ch = kr["lo"], kr["cnt"], kr["child_ptr"], kr["child"]
    assert cnt[0] == len(A) and lo[0] == 0
    for s in range(f["n_states"]):
        kids = ch[cp[s]:cp[s + 1]]
        if len(kids) == 0:
            continue
        own = 1 if f["key_of"][s] >= 0 else 0
        assert lo[kids[0]] == lo[s] + own
        assert (lo[kids][1:] == (lo[kids] + cnt[kids])[:-1]).all()
        assert lo[kids[-1]] + cnt[kids[-1]] == lo[s] + cnt[s]
    assert len(ch) == len(set(ch.tolist()))


# ------------------------------------------------------------------ arguments and states
def test_unbuilt_automata_raise_what_find_all_batch_raises(monkeypatch):
    emul_select.install(monkeypatch)
    A = pkg.flavour("bytes").Automaton()
    for step in ("empty", "trie"):
        with pytest.raises(AttributeError) as want:
            A.find_all_batch([b"a"])
        for name in ("select_batch", "keys_batch", "values_batch", "items_batch"):
            with pytest.raises(AttributeError) as got:
                getattr(A, name)([b"a"])
            assert str(got.value) == str(want.value)
        A.add_word(b"ab", 1)
    A.make_automaton()
    assert A.values_batch([b"a", b"b"]) == [[1], []]
    A.add_word(b"ab", 2)
    with pytest.raises(AttributeError):
        A.values_batch([b"a"])
    A.make_automaton()
    assert A.values_batch([b"a"]) == [[2]]                # values replaced in place are read at call time


def _error(fn):
    try:
        fn()
    except (TypeError, ValueError) as e:
        return type(e), str(e)
    return None


@pytest.mark.parametrize("fl, seq, good, bad, wild, bad_wild", [
    ("bytes", False, b"ab", ["ab", 3], b"?", [b"??", b"", "?"]),
    ("unicode", False, "ab", [b"ab", 3], "?", ["??", "", b"?"]),
    ("bytes", True, (97, 98), [("x",), (-1,), b"ab"], (0,), [(0, 0), (), (70000,)]),
    ("unicode", True, (97, 98), [(1.5,), (2 ** 32,), "ab"], (0,), [(0, 0), (), "a"]),
])
def test_wrong_arguments_raise_the_per_key_errors(fl, seq, good, bad, wild, bad_wild, monkeypatch):
    """the first offending argument decides, in the order keys() checks them: pattern, wildcard, how"""
    emul_select.install(monkeypatch)
    mod = pkg.flavour(fl)
    A = mod.Automaton(mod.STORE_ANY, mod.KEY_SEQUENCE) if seq else mod.Automaton()
    A.add_word(good, 1)
    A.make_automaton()
    names = ("select_batch", "keys_batch", "values_batch", "items_batch")
    cases = []
    for b in bad:
        cases += [((b,), ()), ((b,), (bad_wild[0], 7)), ((good, b), ()), ((good, b), (wild, AT_MOST))]
    for bw in bad_wild:
        cases += [((good,), (bw,)), ((good,), (bw, 7)), ((good, bad[0]), (bw,))]
    cases += [((good,), (wild, 7)), ((good,), (None, -1)), ((good, bad[0]), (wild, 7))]
    for pats, extra in cases:
        want = None
        for p in pats:                                    # what looping keys() raises first
            want = _error(lambda: list(A.keys(p, *extra)))
            if want is not None:
                break
        assert want is not None, (pats, extra)
        for name in names:
            assert _error(lambda: getattr(A, name)(list(pats), *extra)) == want, (name, pats, extra)
    assert A.keys_batch([good], wild, AT_LEAST) == [[good]]


def test_select_host_fails_loudly_without_a_device():
    skip_if_device()
    L = N.lib()
    fake = fake_table()
    pats = np.frombuffer(b"abcd", dtype=np.uint8)
    offs = np.array([0, 2, 4], dtype=np.int64)
    out = np.empty(3, np.int64)
    total = ctypes.c_int64(0)
    assert L.acb_select_host(None, N.ptr(pats), 4, N.ptr(offs), 2, 0, -1, 0, N.ptr(out), None, 0,
                             ctypes.byref(total)) == N.ACB_EINVAL
    A = pkg.flavour("bytes").Automaton()
    A.add_word(b"ab", 1)
    A.make_automaton()
    with pytest.raises(N.NativeError):                    # no CPU fallback behind the Python methods either
        A.keys_batch([b"a"])


def test_deep_wildcards_emulated(monkeypatch):
    emul_select.install(monkeypatch)
    _deep(pkg.flavour("bytes"))


@pytest.mark.gpu
def test_deep_wildcards_gpu():
    _deep(pkg.flavour("bytes"))
    _deep(pkg.flavour("unicode"))


def _deep(mod):
    """patterns with far more wildcard letters than the path the kernel keeps (16 nodes), on keys of up to 60 letters"""
    rng = np.random.default_rng(8)
    wide = mod is pkg.flavour("unicode")
    mk = (lambda s: s) if wide else (lambda s: s.encode())
    A = mod.Automaton(mod.STORE_INTS)
    keys = {"".join(rng.choice(list("ab"), size=int(rng.integers(1, 61)))) for _ in range(150)}
    keys |= {"a" * n for n in range(1, 61)} | {"ab" * 20, "b" + "a" * 40}
    for i, k in enumerate(sorted(keys)):
        A.add_word(mk(k), i)
    A.make_automaton()
    pats = ["?" * n for n in (0, 1, 17, 30, 40, 59, 60, 61)] + ["a" + "?" * 39, "?" * 20 + "a" * 20, "??b" * 14]
    pats = [mk(p) for p in pats]
    for how in HOWS:
        assert A.keys_batch(pats, mk("?"), how) == [list(A.keys(p, mk("?"), how)) for p in pats], how


# ------------------------------------------------------------------ GPU only
@pytest.mark.gpu
def test_all_256_byte_values_on_edges():
    A = pkg.flavour("bytes").Automaton(pkg.STORE_INTS)
    for b in range(256):
        A.add_word(bytes([b, 0x71]), b)
    A.add_word(b"\x00\x00\x00", 1000)
    A.add_word(b"\xff\x00", 1001)
    A.make_automaton()
    assert A.flat()["n_classes"] == 256
    pats = [bytes([b]) for b in range(256)] + [b"\x00\x00", b"", b"\x00?", b"?\x00", b"??", b"???", b"?q"]
    for w in (None, b"?", b"\x00"):
        for how in HOWS:
            assert A.values_batch(pats, w, how) == [list(A.values(p, w, how)) for p in pats], (w, how)


@pytest.mark.gpu
def test_wide_letters_whose_siblings_differ_in_low_bytes():
    S = pkg.flavour("bytes").Automaton(pkg.STORE_ANY, pkg.KEY_SEQUENCE)
    U = pkg.flavour("unicode").Automaton()
    seq_keys = [(0x61, 0x162), (0x61, 0x62), (0x61, 0x6162, 0x62), (0x161,), (0x61, 0x262, 0x62), (0x61, 0x162, 0x63)]
    uni_keys = ["aŢ", "ab", "a\U00010062b", "š", "a\U00020162b", "aŢc", "aŢţ"]
    for A, keys, w in ((S, seq_keys, (0x62,)), (U, uni_keys, "b")):
        for i, k in enumerate(keys):
            A.add_word(k, i)
        A.remove_word(keys[1])
        A.add_word(keys[1], 50)
        A.make_automaton()
        pats = list(keys) + ([(0x61, 0x62), (0x62, 0x62), (0x61, 0x62, 0x62), (0x62,), ()] if A is S else
                             ["ab", "bb", "abb", "b", "", "aŢb", "Ţ"])
        for ww in (None, w):
            for how in HOWS:
                assert A.items_batch(pats, ww, how) == [list(A.items(p, ww, how)) for p in pats], (ww, how)


@pytest.mark.gpu
def test_load_with_a_flat_table_cache_hit(tmp_path):
    mod = pkg.flavour("unicode")
    A = mod.Automaton(mod.STORE_INTS)
    rng = np.random.default_rng(6)
    words = {"".join(rng.choice(list("abcł"), size=int(rng.integers(1, 7)))) for _ in range(300)}
    for i, w in enumerate(sorted(words)):
        A.add_word(w, i)
    for w in sorted(words)[::5]:
        A.remove_word(w)
    A.make_automaton()
    p = str(tmp_path / "a.bin")
    A.save(p)
    B1 = mod.load(p, pickle.loads)                        # writes the flat-table cache
    assert os.path.exists(p + ".acb200")
    B2 = mod.load(p, pickle.loads)                        # installs the cached tables
    pats = ["", "a", "ab", "ł", "a?", "??", "?ł?", "abcł", "zz"]
    for B in (B1, B2):
        assert B.kind == pkg.AHOCORASICK
        for w in (None, "?"):
            for how in HOWS:
                assert B.items_batch(pats, w, how) == [list(B.items(q, w, how)) for q in pats], (w, how)


@pytest.mark.gpu
@pytest.mark.parametrize("fl", ["bytes", "unicode"])
def test_cuda_tensors_on_a_side_stream(fl):
    import torch
    rng = np.random.default_rng(4)
    A = pkg.flavour(fl).Automaton(pkg.STORE_INTS)
    L = A._L
    letters = [0x61, 0x62, 0x3F]
    keys = {tuple(int(x) for x in rng.choice(letters[:2], size=int(rng.integers(1, 6)))) for _ in range(40)}
    for i, k in enumerate(sorted(keys)):
        A.add_word(bytes(k) if L == 1 else "".join(map(chr, k)), i)
    A.make_automaton()
    rows = rng.choice(letters, size=(3001, 3)).astype(DT[L])
    host = np.ascontiguousarray(rows.view(np.uint8).reshape(3001, -1))
    d = torch.from_numpy(host).cuda()
    w = b"?" if L == 1 else "?"
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    for t, h in ((d, host), (d[1:], host[1:])):
        for how in HOWS:
            with torch.cuda.stream(side):
                offs, kid = A.select_batch(t, w, how)
                assert offs.is_cuda and kid.is_cuda and offs.dtype == torch.int64 and kid.dtype == torch.int32
                got = A.keys_batch(t, w, how)
            side.synchronize()
            objs = [r.tobytes() if L == 1 else r.tobytes().decode("utf-32-le") for r in h]
            want = [list(A.keys(p, w, how)) for p in objs]
            assert got == want
            ko = A._key_objs
            o, k = offs.cpu().tolist(), kid.cpu().tolist()
            assert [[ko[x] for x in k[o[i]:o[i + 1]]] for i in range(len(objs))] == want


@pytest.fixture(scope="module")
def published():
    words = [w.encode() for w in published_words(1_000_000)]
    A = pkg.flavour("bytes").Automaton(pkg.STORE_INTS)
    for i, w in enumerate(words):
        A.add_word(w, i)
    A.make_automaton()
    return A, words


@pytest.mark.gpu
def test_output_past_2_31_ids(published):
    """2 200 empty-prefix queries on the 1 M-word key set: 2.2 G ids, checked on the device against the key order"""
    import torch
    A, words = published
    n = 2200
    d = torch.zeros((n, 0), dtype=torch.uint8, device="cuda")
    offs, kid = A.select_batch(d)
    assert int(offs[-1]) == n * len(words) > 2 ** 31
    order = torch.from_numpy(A.key_ranges()["order"]).cuda()
    assert (offs == torch.arange(n + 1, device="cuda", dtype=torch.int64) * len(words)).all()
    rng = np.random.default_rng(1)
    for i in rng.integers(0, n, size=12).tolist() + [0, n - 1]:
        assert torch.equal(kid[i * len(words):(i + 1) * len(words)], order), i
    del kid


@pytest.mark.gpu
def test_published_shape_prefix_and_wildcard_queries(published):
    """1 M prefix queries of 1-3 letters and wildcard patterns on the 1 M-word key set; every slice checked to be one run
    of the key order holding as many keys as start with its prefix, a sample against the per-key method"""
    A, words = published
    rng = np.random.default_rng(7)
    chars = np.frombuffer((string.ascii_letters + string.digits).encode(), dtype=np.uint8)
    n = 1_000_000
    lens = np.full(n, 3)                                  # output within reach: 1 000 of 1 letter (16 k keys each),
    lens[rng.permutation(n)[:201_000]] = 2                # 200 000 of 2 letters, the rest of 3
    lens[rng.permutation(n)[:1000]] = 1
    pats = [bytes(rng.choice(chars, size=int(k))) for k in lens]
    offs, kid = A.select_batch(pats)
    order = A.key_ranges()["order"]
    rank = np.empty(len(order), dtype=np.int64)
    rank[order] = np.arange(len(order))
    srt = sorted(words)
    import bisect
    want_cnt = np.array([bisect.bisect_left(srt, p + b"\x7f") - bisect.bisect_left(srt, p) for p in pats])
    assert (np.diff(offs) == want_cnt).all()
    r = rank[kid]                                         # every slice is one run of the key order
    inner = np.ones(len(kid), dtype=bool)
    inner[offs[:-1][want_cnt > 0]] = False
    assert (np.diff(r)[inner[1:]] == 1).all()
    for i in rng.integers(0, n, size=2000).tolist():
        assert all(words[k].startswith(pats[i]) for k in kid[offs[i]:offs[i + 1]]), i
    for i in rng.integers(0, n, size=4).tolist():           # a per-key call walks all 1 M keys in Python: seconds each
        assert A.values_batch([pats[i]])[0] == list(A.values(pats[i])), i
    wpats = [bytes(rng.choice(chars, size=3)) + b"??" for _ in range(2000)] + [b"?" * 4 + bytes(rng.choice(chars, size=1)) for _ in range(50)]
    for how in HOWS:
        got = A.values_batch(wpats, b"?", how)
        for i in rng.integers(0, len(wpats), size=3).tolist() + [len(wpats) - 1]:
            assert got[i] == list(A.values(wpats[i], b"?", how)), (i, how)
