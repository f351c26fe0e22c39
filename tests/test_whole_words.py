"""whole_words on find_all_batch / find_leftmost_longest_batch / Replacer.replace_batch, filtered on the GPU
(acb_word_filter_device and the acb_*_words host routes).

The answer is always the definition (emul_words.definition) over the full list of the C oracle (per-haystack iter()),
followed by emul_leftmost.greedy and emul_replace.definition for the other two methods; at scale, the numpy restatement
of the same rule (emul_words.flags) over find_all_batch's records.  The CPU tests run the Python layer on the numpy
restatement of the device steps (tests/emul_words.py); the gpu-marked tests run the real kernels."""
import ctypes
import re

import numpy as np
import pytest

import emul
import emul_leftmost
import emul_replace
import emul_words
import pyahocorasick_b200 as pkg
from batch_cases import (CASES, DT, automaton, check_device_capacities, check_host_capacities, fake_table, forms,
                         got_values, key_len, np_greedy, obj, oracle_full, rows, skip_if_device, split, table_and_batch)
from pyahocorasick_b200 import _native as N
from pyahocorasick_b200.automaton import _word_bits

FUZZ_CASES = ["bytes", "latin1", "wide", "mixed"]
SPACE, UNDERSCORE = 0x20, 0x5F


def _is_word(case, words):
    """the word-letter predicate over letter values for a whole_words argument"""
    bytes_fl = CASES[case][0] == "bytes"
    if words is True:
        if bytes_fl:
            return lambda v: re.fullmatch(rb"\w", bytes([v])) is not None
        return lambda v: re.fullmatch(r"\w", chr(v)) is not None
    s = set(words) if bytes_fl else set(map(ord, words))
    return lambda v: v in s


def _word_sets(case):
    if CASES[case][0] == "bytes":
        return [True, b"", b"a_ "]
    return [True, "", "ał_\U0001F600"]


def _random_case(case, rng):
    """keys and haystacks over the case's alphabet plus a space (never a word letter) and an underscore (always one, but
    for the custom sets), so keys begin and end with word and non-word letters"""
    al = CASES[case][2] + [SPACE, UNDERSCORE]
    keys = sorted({tuple(int(x) for x in rng.choice(al, size=int(rng.integers(1, 5)))) for _ in range(int(rng.integers(1, 9)))})
    hays = []
    for _ in range(int(rng.integers(1, 10))):
        r = int(rng.integers(0, 6))
        if r == 0:
            hays.append([])
        elif r == 1:
            hays.append(list(keys[int(rng.integers(0, len(keys)))]))                # one key, matched at both edges
        else:
            hays.append([int(x) for x in rng.choice(al, size=int(rng.integers(1, 40)))])
    if case == "mixed" and all(max(h, default=0) < 256 for h in hays):
        hays.append([0x1F600, 0x61, SPACE, 0x62])
    return keys, hays


def _want(O, keys, hays, case, words):
    """(find_all, leftmost-longest) by the definition over the oracle's full list"""
    kl = [len(k) for k in keys]
    kept = emul_words.definition(hays, oracle_full(O, hays, case), kl, _is_word(case, words))
    return kept, emul_leftmost.greedy(kept, kl)


def _want_replaced(hays, chosen, keys, reps):
    kl = [len(k) for k in keys]
    return [emul_replace.definition(h, [(e, k) for hh, e, k in chosen if hh == i], kl, reps) for i, h in enumerate(hays)]


def _reps(keys):
    return [[0x5A] * (len(k) % 3) for k in keys]          # "", "Z" or "ZZ": latin-1, so the latin-1 table exists


def _check_case(case, keys, hays, words, algo="auto"):
    fl, seq, _ = CASES[case]
    A, O = automaton(fl, seq, keys)
    want_all, want_ll = _want(O, keys, hays, case, words)
    for form, batch in forms([obj(fl, seq, h) for h in hays], hays, A._L, case in ("latin1", "mixed")):
        assert got_values(A.find_all_batch(batch, algo=algo, whole_words=words)) == want_all, (case, form, keys, hays, words)
        assert got_values(A.find_leftmost_longest_batch(batch, algo=algo, whole_words=words)) == want_ll, (case, form, keys, hays, words)
    reps = _reps(keys)
    R = A.replacer({obj(fl, seq, k): obj(fl, seq, r) for k, r in zip(keys, reps)})
    got = R.replace_batch([obj(fl, seq, h) for h in hays], algo=algo, whole_words=words)
    assert got == [obj(fl, seq, h) for h in _want_replaced(hays, want_ll, keys, reps)], (case, keys, hays, words)


# ------------------------------------------------------------------ the word sets
def test_default_sets_equal_re_w():
    bits, n = _word_bits(("bytes", None), 1)
    got = np.unpackbits(bits.view(np.uint8), bitorder="little")[:256]
    got = np.pad(got, (0, 256 - got.size))
    assert [bool(x) for x in got] == [re.fullmatch(rb"\w", bytes([b])) is not None for b in range(256)]
    bits, n = _word_bits(("unicode", None), 4)
    got = np.zeros(0x110000, dtype=bool)
    got[:n] = np.unpackbits(bits.view(np.uint8), bitorder="little")[:n].astype(bool)
    want = np.fromiter((re.fullmatch(r"\w", chr(c)) is not None for c in range(0x110000)), dtype=bool, count=0x110000)
    assert np.array_equal(got, want)
    bits1, n1 = _word_bits(("unicode", None), 1)                  # the latin-1 automaton: the first 256 code points
    got1 = np.zeros(256, dtype=bool)
    got1[:n1] = np.unpackbits(bits1.view(np.uint8), bitorder="little")[:n1].astype(bool)
    assert np.array_equal(got1, want[:256])


def test_empty_and_custom_sets():
    assert _word_bits(("bytes", b""), 1)[1] == 0 and _word_bits(("unicode", ""), 4)[1] == 0
    bits, n = _word_bits(("unicode", "ał"), 1)                # letters at or above 256 leave the latin-1 set
    assert n == 0x62 and bits.size == 4
    bits, n = _word_bits(("unicode", "\U0010FFFF"), 4)
    assert n == 0x110000 and bits[-1] == 1 << 31


# ------------------------------------------------------------------ the Python layer on the restatement (CPU)
def test_restatement_flags_and_compaction():
    rng = np.random.default_rng(1)
    flat = rng.choice(np.frombuffer(b"ab _", dtype=np.uint8), size=400)
    offs = np.array([0, 100, 100, 250, 400], dtype=np.int64)
    hays = [flat[offs[i]:offs[i + 1]].tolist() for i in range(4)]
    key_len = np.array([1, 2, 3])
    full = [(h, e, k) for h in range(4) for e in range(len(hays[h])) for k in range(3) if e - key_len[k] + 1 >= 0]
    bits, n_bits = _word_bits(("bytes", None), 1)
    f = emul_words.flags(flat, offs, 0, 1, np.array(full), key_len, bits, n_bits)
    want = emul_words.definition(hays, full, key_len, _is_word("bytes", True))
    for cap in (0, 1, len(want) - 1, len(want), len(full)):
        stored, count = emul_words.compact(np.array(full), f, cap)
        assert count == len(want) and [tuple(r) for r in stored.tolist()] == want[:cap]
    stored, count = emul_words.compact(np.array(full), f, 7, count=5)
    assert count == 5 + len(want) and [tuple(r) for r in stored.tolist()] == want[:2]


def test_python_layer_on_the_restatement(monkeypatch):
    emul_words.install(monkeypatch)
    rng = np.random.default_rng(17)
    for case in FUZZ_CASES:
        for _ in range(8):
            keys, hays = _random_case(case, rng)
            for words in _word_sets(case):
                _check_case(case, keys, hays, words)


def test_empty_set_equals_no_option(monkeypatch):
    emul.install(monkeypatch)
    emul_leftmost.install(monkeypatch)
    emul_words.install(monkeypatch)
    rng = np.random.default_rng(23)
    for case in FUZZ_CASES:
        keys, hays = _random_case(case, rng)
        A, _ = automaton(*CASES[case][:2], keys)
        batch = [obj(*CASES[case][:2], h) for h in hays]
        for sort in (True, False):
            a, b = A.find_all_batch(batch, sort=sort), A.find_all_batch(batch, sort=sort, whole_words=_word_sets(case)[1])
            assert (got_values(a) == got_values(b)) if sort else sorted(got_values(a)) == sorted(got_values(b))   # unsorted: any order
        assert got_values(A.find_leftmost_longest_batch(batch)) == got_values(A.find_leftmost_longest_batch(batch, whole_words=_word_sets(case)[1]))


def _bytes_automaton(keys, cls_args=()):
    mod = pkg.flavour("bytes")
    A = mod.Automaton(*cls_args)
    for k in keys:
        A.add_word(k, k)
    A.make_automaton()
    return A


def test_worked_examples(monkeypatch):
    emul_leftmost.install(monkeypatch)
    emul_words.install(monkeypatch)
    A = _bytes_automaton([b"new", b"new york"])
    assert list(A.find_leftmost_longest_batch([b"new yorker"], whole_words=True)) == [(0, 2, b"new")]
    assert list(A.find_leftmost_longest_batch([b"new yorker"])) == [(0, 7, b"new york")]
    assert A.replacer({b"new": b"NEW", b"new york": b"NY"}).replace_batch([b"new yorker", b"new york!"], whole_words=True) == \
        [b"NEW yorker", b"NY!"]
    A = _bytes_automaton([b"he", b"hers", b"she"])
    assert list(A.find_all_batch([b"ushers he"], whole_words=True)) == [(0, 8, b"he")]
    R = A.replacer({b"he": b"X", b"hers": b"Y", b"she": b"Z"})
    assert R.replace_batch([b"ushers he"], whole_words=True) == [b"ushers X"]
    # a fixed-stride array: row 0 ends in the key and row 1 starts with a word letter; rows are separate haystacks
    A = _bytes_automaton([b"ab"])
    rows = np.frombuffer(b"x ab" b"abxx" b"ab x" b"xxab", dtype=np.uint8).reshape(4, 4).copy()
    assert list(A.find_all_batch(rows, whole_words=True)) == [(0, 3, b"ab"), (2, 1, b"ab")]
    # UTF-8: with the default set b"caf" is a whole word in b"caf\xc3\xa9"; with bytes 0x80-0xFF as word letters it is not
    A = _bytes_automaton([b"caf"])
    utf8 = bytes(range(0x30, 0x3A)) + bytes(range(0x41, 0x5B)) + bytes(range(0x61, 0x7B)) + b"_" + bytes(range(0x80, 0x100))
    assert list(A.find_all_batch(["café caf".encode()], whole_words=True)) == [(0, 2, b"caf"), (0, 8, b"caf")]
    assert list(A.find_all_batch(["café caf".encode()], whole_words=utf8)) == [(0, 8, b"caf")]
    # keys that are not words themselves
    A = _bytes_automaton([b"#tag", b"foo bar"])
    assert list(A.find_all_batch([b"a #tag, foo bar.", b"x#tag foo barn"], whole_words=True)) == [(0, 5, b"#tag"), (0, 14, b"foo bar")]


def test_set_beyond_latin1_on_a_latin1_batch(monkeypatch):
    emul_words.install(monkeypatch)
    keys = [[0x61], [0xE9, 0x61]]
    hays = [[0x61, 0xE9, 0x61, 0x62], [0x62, 0x61], [0x61]]
    for words in ("bł", "é", "ł\U0001F600"):
        _check_case("latin1", keys, hays, words)


def test_refusals():
    A = _bytes_automaton([b"ab"])
    with pytest.raises(ValueError):
        A.find_all_batch([b"ab"], whole_words=True, ignore_white_space=True)
    with pytest.raises(ValueError):
        A.find_all_batch([b"ab"], whole_words=True, algo="long")
    with pytest.raises(ValueError):
        A.find_long_batch([b"ab"], whole_words=True)
    for bad in ("ab", "", ["a"]):
        with pytest.raises(ValueError if isinstance(bad, str) else TypeError):
            A.find_all_batch([b"ab"], whole_words=bad)
        with pytest.raises(ValueError if isinstance(bad, str) else TypeError):
            A.find_leftmost_longest_batch([b"ab"], whole_words=bad)
        with pytest.raises(ValueError if isinstance(bad, str) else TypeError):
            A.replacer({b"ab": b"x"}).replace_batch([b"ab"], whole_words=bad)
    U = pkg.flavour("unicode").Automaton()
    U.add_word("ab", 1)
    U.make_automaton()
    for bad in (b"ab", b""):
        with pytest.raises(ValueError):
            U.find_all_batch(["ab"], whole_words=bad)
        with pytest.raises(ValueError):
            U.find_leftmost_longest_batch(["ab"], whole_words=bad)
    for fl in ("bytes", "unicode"):
        mod = pkg.flavour(fl)
        S = mod.Automaton(mod.STORE_INTS, mod.KEY_SEQUENCE)
        S.add_word((1, 2), 0)
        S.make_automaton()
        with pytest.raises(ValueError):
            S.find_all_batch([(1, 2)], whole_words=True)
        with pytest.raises(ValueError):
            S.find_leftmost_longest_batch([(1, 2)], whole_words=True)
        with pytest.raises(ValueError):
            S.replacer({(1, 2): (3,)}).replace_batch([(1, 2)], whole_words=True)


def test_c_argument_checks():
    L = N.lib()
    fake = fake_table(1)
    tb = ctypes.addressof(fake)
    n = ctypes.c_int64(0)
    hay = np.frombuffer(b"ab cd ab", dtype=np.uint8).copy()
    offs = np.array([0, 3, 8], dtype=np.int64)
    bits = np.zeros(8, dtype=np.uint32)
    for fn in (L.acb_scan_host_words, L.acb_scan_host_leftmost_words):
        extra = (1,) if fn is L.acb_scan_host_words else ()
        call = lambda t, o, nb, b, algo: fn(t, N.ptr(hay), 8, o, 2, 0, b, nb, None, 8, ctypes.byref(n), algo, *extra)
        assert call(None, N.ptr(offs), 256, N.ptr(bits), N.ALGO_AUTO) == N.ACB_EINVAL
        assert call(tb, N.ptr(offs), 257, N.ptr(bits), N.ALGO_AUTO) == N.ACB_EINVAL                 # n_bits too large
        assert call(tb, N.ptr(offs), -1, N.ptr(bits), N.ALGO_AUTO) == N.ACB_EINVAL
        assert call(tb, N.ptr(offs), 8, None, N.ALGO_AUTO) == N.ACB_EINVAL                          # bits missing
        assert call(tb, N.ptr(offs), 256, N.ptr(bits), N.ALGO_LONG) == N.ACB_EINVAL
        bad = np.array([0, 5, 3], dtype=np.int64)
        assert call(tb, N.ptr(bad), 256, N.ptr(bits), N.ALGO_AUTO) == N.ACB_EINVAL                  # bad offsets
        assert fn(tb, N.ptr(hay), 8, None, 3, 3, N.ptr(bits), 256, None, 8, ctypes.byref(n), N.ALGO_AUTO, *extra) == N.ACB_EINVAL
        assert fn(tb, N.ptr(hay), 8, N.ptr(offs), 2, 0, N.ptr(bits), 256, None, -1, ctypes.byref(n), N.ALGO_AUTO, *extra) == N.ACB_EINVAL
    oo = np.zeros(3, dtype=np.int64)
    total = ctypes.c_int64(0)
    assert L.acb_replace_host_words(None, tb, N.ptr(hay), 8, N.ptr(offs), 2, 0, N.ptr(bits), 256, N.ALGO_AUTO, N.ptr(oo), None, 0,
                                    ctypes.byref(total)) == N.ACB_EINVAL
    rec = np.zeros((4, 3), dtype=np.int32)
    cnt = np.zeros(1, dtype=np.int64)
    dev = lambda t, nb, b, n_rec, cap=4, out=N.ptr(rec), count=N.ptr(cnt): L.acb_word_filter_device(
        t, N.ptr(hay), 8, N.ptr(offs), 2, 0, N.ptr(rec), n_rec, b, nb, out, cap, count, None)
    assert dev(None, 256, N.ptr(bits), 1) == N.ACB_EINVAL
    assert dev(tb, 257, N.ptr(bits), 1) == N.ACB_EINVAL
    assert dev(tb, 9, None, 1) == N.ACB_EINVAL
    assert dev(tb, 256, N.ptr(bits), 1, count=None) == N.ACB_EINVAL
    assert dev(tb, 256, N.ptr(bits), 1, out=None) == N.ACB_EINVAL
    assert dev(tb, 256, N.ptr(bits), -1) == N.ACB_EINVAL
    assert dev(tb, 256, N.ptr(bits), 1 << 31) == N.ACB_ERANGE
    assert dev(tb, 0, None, 0) == N.ACB_OK                                # nothing to filter: no device needed
    for width, most in ((2, 65536), (4, 0x110000)):
        wide = fake_table(width)
        big = np.zeros(most // 32, dtype=np.uint32)
        assert dev(ctypes.addressof(wide), most, N.ptr(big), 0) == N.ACB_OK
        assert dev(ctypes.addressof(wide), most + 1, N.ptr(big), 0) == N.ACB_EINVAL
    ms = ctypes.c_float(1.0)
    assert L.acb_last_words_ms(None) == N.ACB_EINVAL and L.acb_last_words_ms(ctypes.byref(ms)) == N.ACB_OK


def test_host_routes_fail_loudly_without_a_device():
    skip_if_device()
    fake = fake_table(1)
    n = ctypes.c_int64(0)
    hay = np.frombuffer(b"abcd" * 4, dtype=np.uint8)
    offs = np.array([0, 8, 16], dtype=np.int64)
    L = N.lib()
    assert L.acb_scan_host_words(ctypes.addressof(fake), N.ptr(hay), 16, N.ptr(offs), 2, 0, None, 0, None, 8, ctypes.byref(n),
                                 N.ALGO_AUTO, 1) == N.ACB_ECUDA
    assert N.last_error()
    assert L.acb_scan_host_leftmost_words(ctypes.addressof(fake), N.ptr(hay), 16, N.ptr(offs), 2, 0, None, 0, None, 8,
                                          ctypes.byref(n), N.ALGO_AUTO) == N.ACB_ECUDA


# ------------------------------------------------------------------ the real kernels
def _kept_np(A, flat, offs, stride, full, words, width=None):
    """the definition at scale: emul_words.flags over find_all_batch's records"""
    L = A._L if width is None else width
    bits, n_bits = _word_bits(A._words(words), L)
    raw = rows(full)
    return raw[emul_words.flags(flat, offs, stride, L, raw, key_len(A), bits, n_bits)]


@pytest.mark.gpu
@pytest.mark.parametrize("algo", ["filter", "dfa"])
def test_gpu_fuzz_against_the_definition(algo):
    rng = np.random.default_rng(31)
    for case in FUZZ_CASES:
        for _ in range(5):
            keys, hays = _random_case(case, rng)
            for words in _word_sets(case):
                _check_case(case, keys, hays, words, algo)


@pytest.mark.gpu
def test_gpu_worked_examples():
    A = _bytes_automaton([b"new", b"new york"])
    assert list(A.find_leftmost_longest_batch([b"new yorker"], whole_words=True)) == [(0, 2, b"new")]
    A = _bytes_automaton([b"he", b"hers", b"she"])
    assert list(A.find_all_batch([b"ushers he"], whole_words=True)) == [(0, 8, b"he")]
    A = _bytes_automaton([b"ab"])
    rows = np.frombuffer(b"x ab" b"abxx" b"ab x" b"xxab", dtype=np.uint8).reshape(4, 4).copy()
    assert list(A.find_all_batch(rows, whole_words=True)) == [(0, 3, b"ab"), (2, 1, b"ab")]


@pytest.mark.gpu
@pytest.mark.parametrize("fl", ["bytes", "unicode"])
def test_gpu_cuda_tensors_on_a_side_stream(fl):
    import torch
    rng = np.random.default_rng(5)
    case = "bytes" if fl == "bytes" else "wide"
    al = CASES[case][2][:2] + [SPACE]
    keys = [list(k) for k in {tuple(int(x) for x in rng.choice(al, size=int(rng.integers(1, 5)))) for _ in range(12)}]
    A, O = automaton(*CASES[case][:2], keys)
    L = A._L
    hays = [[int(x) for x in rng.choice(al, size=7)] for _ in range(300)]
    host = np.stack([np.asarray(h, dtype=DT[L]).view(np.uint8) for h in hays])
    d = torch.from_numpy(host).cuda()
    views = {"whole": (d, hays)}
    if L == 1:
        views["misaligned"] = (d[1:], hays[1:])
        assert d[1:].data_ptr() % 16 != 0
    reps = _reps(keys)
    R = A.replacer({obj(*CASES[case][:2], k): obj(*CASES[case][:2], r) for k, r in zip(keys, reps)})
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    for words in (True, _word_sets(case)[1]):
        assert got_values(A.find_all_batch(host, whole_words=words)) == _want(O, keys, hays, case, words)[0]
        for name, (t, hs) in views.items():
            want_all, want_ll = _want(O, keys, hs, case, words)
            with torch.cuda.stream(side):
                m_all = A.find_all_batch(t, whole_words=words)
                m_ll = A.find_leftmost_longest_batch(t, whole_words=words)
                flat, offs = R.replace_batch(t, whole_words=words)
                side.synchronize()
            assert got_values(m_all) == want_all, (name, words)
            assert got_values(m_ll) == want_ll, (name, words)
            got = split(flat.cpu().numpy(), offs.cpu().numpy(), L)
            assert got == _want_replaced(hs, want_ll, keys, reps), (name, words)


@pytest.mark.gpu
def test_gpu_exact_counts_at_every_capacity():
    import torch
    keys = [b"a", b"ab", b"ba", b"aba", b"b b"]
    A = _bytes_automaton(keys)
    hays = [b"ab ba aba abab b b a" * 20, b"", b"a", b"ab_ab ba-ba"]
    L = N.lib()
    tb, flat, offs = table_and_batch(A, hays)
    bits, n_bits = _word_bits(("bytes", None), 1)
    batch = (tb, N.ptr(flat), flat.size, N.ptr(offs), len(hays), 0, N.ptr(bits), n_bits)
    for leftmost in (False, True):
        want = rows(A.find_leftmost_longest_batch(hays, whole_words=True) if leftmost else A.find_all_batch(hays, whole_words=True))
        assert len(want) > 10
        if leftmost:
            check_host_capacities(lambda out, cap, found: L.acb_scan_host_leftmost_words(*batch, out, cap, found, N.ALGO_AUTO), want)
        else:
            check_host_capacities(lambda out, cap, found: L.acb_scan_host_words(*batch, out, cap, found, N.ALGO_AUTO, 1), want)
    # the replacement: the exact output size past out_cap
    R = A.replacer({k: k.upper() + b"!" for k in keys})
    want = R.replace_batch(hays, whole_words=True)
    r = R._replacer(tb, False, 0)
    total = ctypes.c_int64(0)
    oo = np.empty(len(hays) + 1, dtype=np.int64)
    size = sum(map(len, want))
    for cap in (0, 1, size - 1, size):
        out = np.zeros(max(cap, 1), dtype=np.uint8)
        rc = L.acb_replace_host_words(r, tb, N.ptr(flat), flat.size, N.ptr(offs), len(hays), 0, N.ptr(bits), n_bits, N.ALGO_AUTO,
                                      N.ptr(oo), N.ptr(out), cap, ctypes.byref(total))
        assert total.value == size and rc == (N.ACB_OK if cap >= size else N.ACB_EOVERFLOW)
        if cap >= size:
            assert [out[oo[i]:oo[i + 1]].tobytes() for i in range(len(hays))] == want
    # the device entry: any record order
    full = A.find_all_batch(hays)
    rec = rows(full).astype(np.int32)
    rec = rec[np.random.default_rng(0).permutation(len(rec))]
    want = rec[emul_words.flags(flat, offs, 0, 1, rec, key_len(A), bits, n_bits)].astype(np.int64)
    d_rec = torch.from_numpy(np.ascontiguousarray(rec)).cuda()
    d_hay, d_off = torch.from_numpy(flat).cuda(), torch.from_numpy(offs).cuda()
    d_bits = torch.from_numpy(bits.view(np.int32).copy()).cuda()
    check_device_capacities(lambda out, cap, cnt, s: L.acb_word_filter_device(
        tb, d_hay.data_ptr(), flat.size, d_off.data_ptr(), len(hays), 0, d_rec.data_ptr(), len(rec), d_bits.data_ptr(), n_bits,
        out, cap, cnt, s), want, d_rec)


@pytest.mark.gpu
def test_gpu_c2_planted_against_the_definition():
    from pyahocorasick_b200 import synth
    w = synth.make("C2", scale=0.05)
    A = synth.build_automaton(w.keys)
    stride = w.haystacks.shape[1]
    for words in (True, b""):
        for algo in ("filter", "dfa"):
            full = A.find_all_batch(w.haystacks, algo=algo)
            want = _kept_np(A, w.haystacks.reshape(-1), None, stride, full, words)
            assert np.array_equal(rows(A.find_all_batch(w.haystacks, algo=algo, whole_words=words)), want)
            got = rows(A.find_leftmost_longest_batch(w.haystacks, algo=algo, whole_words=words))
            assert np.array_equal(got, np_greedy(np.rec.fromarrays(want.T, names="hay_id,end_index,key_id"), key_len(A)))
        if words == b"":
            assert np.array_equal(rows(A.find_all_batch(w.haystacks, whole_words=b"")), rows(A.find_all_batch(w.haystacks)))
            assert np.array_equal(rows(A.find_leftmost_longest_batch(w.haystacks, whole_words=b"")),
                                  rows(A.find_leftmost_longest_batch(w.haystacks)))


@pytest.mark.gpu
def test_gpu_single_haystack_of_256_mib():
    rng = np.random.default_rng(21)
    keys = sorted({bytes(rng.choice(list(b"ac g"), size=int(rng.integers(3, 7))).tolist()) for _ in range(24)})
    A = _bytes_automaton(keys)
    text = rng.choice(np.frombuffer(b"acg ", dtype=np.uint8), size=256 << 20)
    offs = np.array([0, text.size], dtype=np.int64)
    full = A.find_all_batch((text, offs))
    want = _kept_np(A, text, offs, 0, full, True)
    assert len(want) > 200_000
    assert np.array_equal(rows(A.find_all_batch((text, offs), whole_words=True)), want)
    got = rows(A.find_leftmost_longest_batch((text, offs), whole_words=True))
    assert np.array_equal(got, np_greedy(np.rec.fromarrays(want.T, names="hay_id,end_index,key_id"), key_len(A)))


@pytest.mark.gpu
def test_gpu_batch_past_2_gib():
    """a CUDA tensor of 2^31 + 2^24 bytes in 2 080 rows, keys planted at row edges, after word letters and across 2^31:
    neighbour addresses need 64 bits"""
    import torch
    keys = [b"qzq", b"zqz", b"qzqzx"]
    A = _bytes_automaton(keys)
    n_rows, stride = 2080, ((1 << 31) + (1 << 24)) // 2080 // 16 * 16
    d = torch.randint(0, 16, (n_rows, stride), dtype=torch.uint8, device="cuda")
    d += ord("a")                                                            # a..p: no key letter but for planted ones
    d[:, ::97] = ord(" ")
    rng = np.random.default_rng(2)
    plants = [b" qzqzx ", b" qzq ", b"aqzqzx ", b" zqzb"]
    for r in rng.integers(0, n_rows, size=800).tolist():
        c = int(rng.integers(0, stride - 8))
        p = plants[int(rng.integers(0, len(plants)))]
        d[r, c:c + len(p)] = torch.tensor(list(p), dtype=torch.uint8)
    d[-1, -4:] = torch.tensor(list(b" qzq"), dtype=torch.uint8)         # at the last letter, past 2^31
    d[0, :4] = torch.tensor(list(b"qzq "), dtype=torch.uint8)           # at the first letter
    d[5, -4:] = torch.tensor(list(b" zqz"), dtype=torch.uint8)          # row 6 starts with a word letter
    d[6, :3] = torch.tensor(list(b"qzq"), dtype=torch.uint8)
    full = A.find_all_batch(d)
    raw = rows(full)
    kl = key_len(A)
    flat = d.view(-1)
    start = raw[:, 0] * stride + raw[:, 1] - kl[raw[:, 2]] + 1
    end = raw[:, 0] * stride + raw[:, 1]
    left = np.where(raw[:, 1] - kl[raw[:, 2]] + 1 > 0, start - 1, -1)
    right = np.where(raw[:, 1] + 1 < stride, end + 1, -1)

    def letters(idx):
        v = np.full(len(idx), ord(" "), dtype=np.int64)
        ok = idx >= 0
        v[ok] = flat[torch.from_numpy(idx[ok]).cuda()].cpu().numpy()
        return v
    word = lambda v: np.array([re.fullmatch(rb"\w", bytes([int(x)])) is not None for x in range(256)])[v]
    want = raw[~word(letters(left)) & ~word(letters(right))]
    got = A.find_all_batch(d, whole_words=True)
    assert n_rows * stride > (1 << 31) and len(want) > 300 and len(want) < len(raw)
    assert (want[:, 0] * stride + want[:, 1] >= (1 << 31)).any()
    assert np.array_equal(rows(got), want)
    ll = A.find_leftmost_longest_batch(d, whole_words=True)
    assert np.array_equal(rows(ll), np_greedy(np.rec.fromarrays(want.T, names="hay_id,end_index,key_id"), kl))


@pytest.mark.gpu
def test_gpu_four_byte_bitmap_near_the_last_code_point():
    import torch
    U = pkg.flavour("unicode").Automaton()
    U.add_word("a", "a")
    U.add_word("\U0010FFFDa", "Xa")
    U.make_automaton()
    hays = ["a\U0010FFFF", "\U0010FFFEa", "a", "\U0010FFFDa\U0010FFFE", "éa"]
    words = "\U0010FFFFé"                               # n_bits = 0x110000
    assert _word_bits(("unicode", words), 4)[1] == 0x110000
    want = [(1, 1, "a"), (2, 0, "a"), (3, 1, "Xa"), (3, 1, "a")]
    assert list(U.find_all_batch(hays, whole_words=words)) == want
    assert list(U.find_leftmost_longest_batch(hays, whole_words=words)) == [(1, 1, "a"), (2, 0, "a"), (3, 1, "Xa")]
    assert U.replacer({"a": "b", "\U0010FFFDa": "c"}).replace_batch(hays, whole_words=words) == \
        ["a\U0010FFFF", "\U0010FFFEb", "b", "c\U0010FFFE", "éa"]
    rows = np.stack([np.array([ord(c) for c in h.ljust(3, " ")], dtype="<u4").view(np.uint8) for h in hays])
    got = U.find_all_batch(torch.from_numpy(rows).cuda(), whole_words=words)
    assert list(got) == want


@pytest.mark.gpu
def test_gpu_launch_counts_of_the_host_routes():
    import test_host_route_launches as hr
    from pyahocorasick_b200 import synth
    A = synth.build_automaton(hr.KEYS)
    L = N.lib()
    tb = A._ensure_table(0)
    flat, off = hr._batch()
    bits, n_bits = _word_bits(("bytes", None), 1)
    batch = (tb, N.ptr(flat), flat.size, N.ptr(off), len(off) - 1, 0, N.ptr(bits), n_bits)
    FILTER = 1 + 2                                                 # flags, emit + count
    routes = {
        "scan": (lambda: hr._records(L, lambda out, n: L.acb_scan_host_words(*batch, out, hr.CAP, n, N.ALGO_FILTER, 1)), 1 + FILTER + 1),
        "leftmost": (lambda: hr._records(L, lambda out, n: L.acb_scan_host_leftmost_words(*batch, out, hr.CAP, n, N.ALGO_FILTER)),
                     1 + FILTER + hr.SELECTION),
        "replace": (lambda: hr._with_replacer(L, tb, lambda r, oo, o, oc, t: L.acb_replace_host_words(
            r, *batch, N.ALGO_FILTER, oo, o, oc, t)), 1 + FILTER + hr.SELECTION + hr.REPLACEMENT),
    }
    for name, (run, want) in routes.items():
        run()
        before = L.acb_launch_count()
        run()
        assert L.acb_launch_count() - before == want, name
