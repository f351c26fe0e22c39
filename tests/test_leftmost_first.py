"""find_leftmost_first_batch / acb_leftmost_first_device / acb_scan_host_leftmost_kind and leftmost-first replacers:
leftmost-first non-overlapping matches (priority by key order) selected on the GPU from the full match list.

Two answers stand against each other: the definition (emul_leftmost_first.greedy_first) over the C oracle's full list,
and Python's `re` (tests/first_cases.py), whose alternation is leftmost-first by its own rules.  The CPU tests run the
numpy restatement of the device steps at tiny tile sizes; the gpu-marked tests run the real kernels."""
import ctypes
import pickle

import numpy as np
import pytest

import emul_leftmost_first as elf
import emul_words
import first_cases
import pyahocorasick_b200 as pkg
from batch_cases import (CASES, DT, automaton, check_device_capacities, check_host_capacities, fake_table, forms,
                         got_values, key_len, leftmost_random_case, leftmost_structured_cases, obj, oracle_full, replace_reps,
                         rows, skip_if_device, split, table_and_batch)
from pyahocorasick_b200 import _native as N
from pyahocorasick_b200.automaton import _word_bits

TILES = [1, 2, 3, 7]
TEXT_CASES = ("bytes", "latin1", "wide", "mixed")


def _want(O, keys, hays, case="bytes"):
    return elf.greedy_first(oracle_full(O, hays, case), [len(k) for k in keys])


def _word_letters(case, rng):
    """a random explicit word set over the case's alphabet (and the no-match letter c): (letters, whole_words argument)"""
    fl = CASES[case][0]
    al = CASES[case][2] + [0x63]
    pick = [c for c in al if rng.integers(0, 2)]
    arg = bytes(pick) if fl == "bytes" else "".join(map(chr, pick))
    return pick, arg


def runs_cases(W):
    """keys a^1 .. a^W added shortest-first and longest-first, on runs of a of every length up to 3W + 1"""
    a = 0x61
    hays = [[a] * r + [0x62] for r in range(1, 3 * W + 2)]
    hays.append(sum(hays, []))
    for order in (range(1, W + 1), range(W, 0, -1)):
        yield [[a] * k for k in order], hays


# ------------------------------------------------------------------ the definition, `re` and the restatement (CPU)
def test_the_documented_examples():
    keys = [b"sam", b"samwise"]
    A, O = automaton("bytes", False, [list(k) for k in keys])
    assert _want(O, [list(k) for k in keys], [list(b"samwise gamgee")]) == [(0, 2, 0)]
    assert first_cases.find("bytes", [list(k) for k in keys], [list(b"samwise gamgee")]) == [(0, 2, 0)]
    keys = [list(b"b"), list(b"abcd")]
    _, O = automaton("bytes", False, keys)
    assert _want(O, keys, [list(b"abcd")]) == [(0, 3, 1)]               # leftmost beats priority
    assert first_cases.find("bytes", keys, [list(b"abcd")]) == [(0, 3, 1)]


def test_definition_agrees_with_re():
    rng = np.random.default_rng(1)
    for case in TEXT_CASES:
        fl, seq, _ = CASES[case]
        for _ in range(40):
            keys, hays = leftmost_random_case(case, rng)
            keys = [list(k) for k in keys]
            rng.shuffle(keys)                                                # priority is not the sorted order
            _, O = automaton(fl, seq, keys)
            full = oracle_full(O, hays, case)
            kl = [len(k) for k in keys]
            assert elf.greedy_first(full, kl) == first_cases.find(case, keys, hays), (case, keys, hays)
            letters, _ = _word_letters(case, rng)
            words = set(letters)
            whole = emul_words.definition(hays, full, kl, lambda v: v in words)
            assert elf.greedy_first(whole, kl) == first_cases.find(case, keys, hays, letters), (case, keys, hays, letters)
    for keys, hays in list(leftmost_structured_cases()) + [c for W in (1, 4, 9) for c in runs_cases(W)]:
        _, O = automaton("bytes", False, keys)
        assert _want(O, keys, hays) == first_cases.find("bytes", keys, hays)


@pytest.mark.parametrize("tile", TILES + [2048])
def test_restatement_equals_the_definition(tile):
    rng = np.random.default_rng(tile)
    for case, (fl, seq, _) in CASES.items():
        for _ in range(12):
            keys, hays = leftmost_random_case(case, rng)
            keys = [list(k) for k in keys]
            rng.shuffle(keys)
            _, O = automaton(fl, seq, keys)
            full = oracle_full(O, hays, case)
            kl = np.array([len(k) for k in keys])
            raw = np.array(full, dtype=np.int64).reshape(-1, 3)
            got = elf.select_first(raw[rng.permutation(len(raw))], kl, int(kl.max()), tile)
            assert [tuple(r) for r in got.tolist()] == elf.greedy_first(full, kl), (case, keys, hays)
    for keys, hays in list(leftmost_structured_cases()) + [c for W in (1, 2, 5, 16) for c in runs_cases(W)]:
        _, O = automaton("bytes", False, keys)
        full = oracle_full(O, hays)
        kl = np.array([len(k) for k in keys])
        got = elf.select_first(np.array(full, dtype=np.int64).reshape(-1, 3), kl, int(kl.max()), tile)
        assert [tuple(r) for r in got.tolist()] == elf.greedy_first(full, kl)


def _check_methods(A, O, case, keys, hays, rng, whole_words=False, letters=None):
    """find_leftmost_first_batch in every input form, replace_batch and a leftmost_first stream batch, against `re`
    (text cases) or the definition (key sequences)"""
    fl, seq, _ = CASES[case]
    kl = [len(k) for k in keys]
    full = oracle_full(O, hays, case)
    if whole_words:
        words = set(letters)
        full = emul_words.definition(hays, full, kl, lambda v: v in words)
    want = elf.greedy_first(full, kl)
    if case in TEXT_CASES:
        assert want == first_cases.find(case, keys, hays, letters if whole_words else None)
    for form, batch in forms([obj(fl, seq, h) for h in hays], hays, A._L, case in ("latin1", "mixed")):
        assert got_values(A.find_leftmost_first_batch(batch, whole_words=whole_words)) == want, (case, form)
    reps = replace_reps(case, keys, rng)
    R = A.replacer({obj(fl, seq, k): obj(fl, seq, r) for k, r in zip(keys, reps)}, leftmost_first=True)
    out = R.replace_batch([obj(fl, seq, h) for h in hays], whole_words=whole_words)
    from emul_replace import definition
    by_hay = [[(e, k) for h, e, k in want if h == i] for i in range(len(hays))]
    expect = [definition(h, c, kl, reps) for h, c in zip(hays, by_hay)]
    assert out == [obj(fl, seq, x) for x in expect], case
    if case in TEXT_CASES:
        assert expect == first_cases.sub(case, keys, reps, hays, letters if whole_words else None)
    B = A.stream_batch(len(hays), leftmost_first=True, whole_words=whole_words)
    got = []
    for lo in range(0, max(map(len, hays), default=0) + 1, 3):
        m = B.feed([obj(fl, seq, h[lo:lo + 3]) for h in hays])
        got += got_values(m)
    got += got_values(B.finish())
    assert sorted(got) == want, case


@pytest.mark.parametrize("tile", [1, 3, 2048])
def test_python_layer_on_the_restatement(monkeypatch, tile):
    elf.install(monkeypatch, tile)
    rng = np.random.default_rng(7 + tile)
    for case, (fl, seq, _) in CASES.items():
        for _ in range(3):
            keys, hays = leftmost_random_case(case, rng)
            keys = [list(k) for k in keys]
            rng.shuffle(keys)
            A, O = automaton(fl, seq, keys)
            _check_methods(A, O, case, keys, hays, rng)
            if not seq:
                letters, _ = _word_letters(case, rng)
                arg = bytes(letters) if fl == "bytes" else "".join(map(chr, letters))
                _check_methods_words(A, O, case, keys, hays, rng, letters, arg)


def _check_methods_words(A, O, case, keys, hays, rng, letters, arg):
    fl, seq, _ = CASES[case]
    kl = [len(k) for k in keys]
    words = set(letters)
    want = elf.greedy_first(emul_words.definition(hays, oracle_full(O, hays, case), kl, lambda v: v in words), kl)
    assert want == first_cases.find(case, keys, hays, letters)
    assert got_values(A.find_leftmost_first_batch([obj(fl, seq, h) for h in hays], whole_words=arg)) == want
    B = A.stream_batch(len(hays), leftmost_first=True, whole_words=arg)
    got = got_values(B.feed([obj(fl, seq, h[:5]) for h in hays]))
    got += got_values(B.feed([obj(fl, seq, h[5:]) for h in hays]))
    got += got_values(B.finish())
    assert sorted(got) == want


def test_priority_follows_insertion(monkeypatch):
    """add_word of a present key keeps its place; remove_word then add_word moves a key to the end; clear starts over;
    a pickle round trip numbers keys afresh, and its priority is the new id order"""
    elf.install(monkeypatch)
    mod = pkg.flavour("bytes")
    A = mod.Automaton()
    for k in (b"sam", b"samwise", b"gamgee"):
        A.add_word(k, k)
    A.add_word(b"sam", b"SAM")                                   # a new value, the same place
    A.make_automaton()
    assert A.find_leftmost_first_batch([b"samwise"]).values() == [b"SAM"]
    A.remove_word(b"sam")
    A.add_word(b"sam", b"sam again")                             # now after samwise
    A.make_automaton()
    assert A.find_leftmost_first_batch([b"samwise"]).values() == [b"samwise"]
    ids = {k: A._key_ids[k] for k in (b"sam", b"samwise", b"gamgee")}
    assert ids[b"sam"] > ids[b"samwise"]                          # a hole at the old id, the key at the end
    B = pickle.loads(pickle.dumps(A))
    order = sorted(B._key_ids, key=B._key_ids.get)
    want = b"samwise" if order.index(b"samwise") < order.index(b"sam") else b"sam again"
    assert B.find_leftmost_first_batch([b"samwise"]).values() == [want]
    A.clear()
    for k in (b"samwise", b"sam"):
        A.add_word(k, k)
    A.make_automaton()
    assert A.find_leftmost_first_batch([b"samwise"]).values() == [b"samwise"]


def test_refusals():
    mod = pkg.flavour("bytes")
    A = mod.Automaton()
    A.add_word(b"ab", 0)
    with pytest.raises(AttributeError):
        A.find_leftmost_first_batch([b"ab"])                     # not built
    A.make_automaton()
    for algo in ("long", "x"):
        with pytest.raises(ValueError):
            A.find_leftmost_first_batch([b"ab"], algo=algo)
    for kw in ({"leftmost_longest": True}, {"long": True}, {"ignore_white_space": True}):
        with pytest.raises(ValueError):
            A.stream_batch(2, leftmost_first=True, **kw)
    S = pkg.flavour("bytes").Automaton(mod.STORE_INTS, mod.KEY_SEQUENCE)
    S.add_word((1, 2), 0)
    S.make_automaton()
    with pytest.raises(ValueError):
        S.find_leftmost_first_batch([(1, 2)], whole_words=True)      # KEY_SEQUENCE has no words
    with pytest.raises(ValueError):
        A.find_leftmost_first_batch([b"ab"], whole_words="ab")       # a word set of the other flavour


def test_c_entry_argument_errors():
    L = N.lib()
    fake = fake_table(1)
    tb = ctypes.addressof(fake)
    n = ctypes.c_int64(0)
    hay = np.zeros(16, dtype=np.uint8)
    cnt = np.zeros(1, dtype=np.int64)
    assert L.acb_leftmost_first_device(None, N.ptr(hay), 1, 1, 16, N.ptr(hay), 1, N.ptr(cnt), None) == N.ACB_EINVAL
    assert L.acb_leftmost_first_device(tb, None, 1, 1, 16, N.ptr(hay), 1, N.ptr(cnt), None) == N.ACB_EINVAL
    assert L.acb_leftmost_first_device(tb, N.ptr(hay), 1, 1, 16, None, 1, N.ptr(cnt), None) == N.ACB_EINVAL
    assert L.acb_leftmost_first_device(tb, N.ptr(hay), 1 << 31, 1, 16, N.ptr(hay), 1, N.ptr(cnt), None) == N.ACB_ERANGE
    args = (N.ptr(hay), 16, None, 1, 16, None, -1, None, 8, ctypes.byref(n), N.ALGO_AUTO)
    assert L.acb_scan_host_leftmost_kind(None, N.SELECT_FIRST, *args) == N.ACB_EINVAL
    assert L.acb_scan_host_leftmost_kind(tb, 2, *args) == N.ACB_EINVAL
    assert L.acb_scan_host_leftmost_kind(tb, N.SELECT_FIRST, N.ptr(hay), 16, None, 1, 16, None, -1, None, 8, ctypes.byref(n),
                                         N.ALGO_LONG) == N.ACB_EINVAL
    assert L.acb_scan_host_leftmost_kind(tb, N.SELECT_FIRST, N.ptr(hay), 16, None, 1, 16, None, 300, None, 8, ctypes.byref(n),
                                         N.ALGO_AUTO) == N.ACB_EINVAL                        # 300 bits need a bitmap
    r = ctypes.c_void_p()
    offs = np.zeros(2, dtype=np.int64)
    assert L.acb_replacer_new_kind(tb, 5, None, 0, N.ptr(offs), 1, ctypes.byref(r)) == N.ACB_EINVAL
    ss = ctypes.c_void_p()
    assert L.acb_streams_new_leftmost_kind(tb, 1, -1, None, -1, ctypes.byref(ss)) == N.ACB_EINVAL
    assert L.acb_streams_new_leftmost_kind(None, 1, N.SELECT_FIRST, None, -1, ctypes.byref(ss)) == N.ACB_EINVAL


def test_host_route_fails_loudly_without_a_device():
    skip_if_device()
    fake = fake_table(1)
    n = ctypes.c_int64(0)
    hay = np.frombuffer(b"abcd" * 4, dtype=np.uint8)
    offs = np.array([0, 8, 16], dtype=np.int64)
    assert N.lib().acb_scan_host_leftmost_kind(ctypes.addressof(fake), N.SELECT_FIRST, N.ptr(hay), 16, N.ptr(offs), 2, 0, None, -1,
                                               None, 8, ctypes.byref(n), N.ALGO_AUTO) == N.ACB_ECUDA
    assert N.last_error()


# ------------------------------------------------------------------ the real kernels
@pytest.mark.gpu
@pytest.mark.parametrize("algo", ["filter", "dfa"])
def test_gpu_fuzz_against_re_and_the_definition(algo):
    rng = np.random.default_rng(11)
    for case, (fl, seq, _) in CASES.items():
        for _ in range(6):
            keys, hays = leftmost_random_case(case, rng)
            keys = [list(k) for k in keys]
            rng.shuffle(keys)
            A, O = automaton(fl, seq, keys)
            want = _want(O, keys, hays, case)
            if case in TEXT_CASES:
                assert want == first_cases.find(case, keys, hays)
            for form, batch in forms([obj(fl, seq, h) for h in hays], hays, A._L, case in ("latin1", "mixed")):
                assert got_values(A.find_leftmost_first_batch(batch, algo=algo)) == want, (case, form, keys, hays)
            if case in TEXT_CASES:
                letters, arg = _word_letters(case, rng)
                got = got_values(A.find_leftmost_first_batch([obj(fl, seq, h) for h in hays], algo=algo, whole_words=arg))
                assert got == first_cases.find(case, keys, hays, letters), (case, keys, hays, letters)
    for keys, hays in list(leftmost_structured_cases()) + [c for W in (1, 3, 16, 64) for c in runs_cases(W)]:
        A, O = automaton("bytes", False, keys)
        assert got_values(A.find_leftmost_first_batch([bytes(h) for h in hays], algo=algo)) == first_cases.find("bytes", keys, hays)


@pytest.mark.gpu
def test_gpu_python_methods_every_case():
    rng = np.random.default_rng(12)
    for case, (fl, seq, _) in CASES.items():
        for _ in range(3):
            keys, hays = leftmost_random_case(case, rng)
            keys = [list(k) for k in keys]
            rng.shuffle(keys)
            A, O = automaton(fl, seq, keys)
            _check_methods(A, O, case, keys, hays, rng)
            if not seq:
                letters, arg = _word_letters(case, rng)
                _check_methods_words(A, O, case, keys, hays, rng, letters, arg)


@pytest.mark.gpu
def test_gpu_runs_over_many_tiles_both_orders():
    """runs of a under a^1 .. a^W (and ab, bababa): added longest-first, leftmost-first is leftmost-longest (W chains
    that never meet); added shortest-first, every candidate in a run is the single letter a"""
    rng = np.random.default_rng(9)
    for W in (1, 3, 16, 64):
        runs = rng.integers(1, 3 * W + 2, size=40000 // W + 2000)
        hay = b"b".join(b"a" * int(r) for r in runs)
        hays = [hay, b"", hay[: len(hay) // 3], b"ab" * 5000]
        every = [b"a" * k for k in range(1, W + 1)] + [b"ab", b"ba" * 3]
        for keys in (sorted(every, key=len, reverse=True), sorted(every, key=len)):
            A, _ = automaton("bytes", False, [list(k) for k in keys])
            got = rows(A.find_leftmost_first_batch(hays))
            full = A.find_all_batch(hays)
            want = np.array(elf.greedy_first(zip(full.hay_id, full.end_index, full.key_id), key_len(A)), dtype=np.int64)
            assert len(want) > 3 * 2048
            assert np.array_equal(got, want), W
            if len(keys[0]) >= len(keys[-1]):                           # longest-first: leftmost-longest
                assert np.array_equal(got, rows(A.find_leftmost_longest_batch(hays)))


@pytest.mark.gpu
def test_gpu_priority_after_removal_duplicates_and_pickle():
    rng = np.random.default_rng(4)
    al = list(b"abc")
    for trial in range(4):
        words = sorted({bytes(rng.choice(al, size=int(rng.integers(1, 6))).tolist()) for _ in range(30)})
        rng.shuffle(words)
        A = pkg.flavour("bytes").Automaton()
        for w in words:
            A.add_word(w, w)
        for w in words[::3]:
            A.add_word(w, w)                                          # duplicates keep their place
        for w in words[1::4]:
            A.remove_word(w)
        for w in words[1::8]:
            A.add_word(w, w)                                          # back, at the end
        A.make_automaton()
        hays = [bytes(rng.choice(al, size=int(rng.integers(0, 200))).tolist()) for _ in range(50)]
        for X in (A, pickle.loads(pickle.dumps(A))):
            order = [k for k in sorted(X._key_ids, key=X._key_ids.get)]
            want = [(h, e, order[k]) for h, e, k in first_cases.find("bytes", [list(k) for k in order], [list(x) for x in hays])]
            got = X.find_leftmost_first_batch(hays)
            assert list(zip(got.hay_id.tolist(), got.end_index.tolist(), got.values())) == want, trial


@pytest.mark.gpu
@pytest.mark.parametrize("bits", [64, 65])
def test_gpu_sort_key_of_64_and_65_bits(bits):
    """acb_leftmost_first_device with max_hay_letters set so that hay | start | key_id takes 64 bits (one radix sort) or
    65 (two stable passes); the records are a real full list in any order"""
    import torch
    rng = np.random.default_rng(bits)
    keys = [list(k) for k in (b"ab", b"abc", b"bca", b"c", b"cab", b"abcab", b"b")]
    rng.shuffle(keys)
    A, O = automaton("bytes", False, keys)
    hays = [bytes(rng.choice(list(b"abc"), size=int(rng.integers(0, 300))).tolist()) for _ in range(200)]
    full = A.find_all_batch(hays)
    rec = np.stack([full.hay_id, full.end_index, full.key_id], axis=1).astype(np.int32)
    rec = rec[rng.permutation(len(rec))]
    want = np.array(elf.greedy_first(rec.tolist(), key_len(A)), dtype=np.int64)
    bh, bk = (len(hays) - 1).bit_length(), (len(keys) - 1).bit_length()
    max_letters = (1 << (bits - bh - bk)) - 1
    assert bh + max_letters.bit_length() + bk == bits
    tb = A._ensure_table(0)
    d_rec = torch.from_numpy(np.ascontiguousarray(rec)).cuda()
    out = torch.empty((len(rec), 3), dtype=torch.int32, device="cuda")
    cnt = torch.zeros(1, dtype=torch.int64, device="cuda")
    N.check(N.lib().acb_leftmost_first_device(tb, d_rec.data_ptr(), len(rec), len(hays), max_letters, out.data_ptr(), len(rec),
                                              cnt.data_ptr(), torch.cuda.current_stream().cuda_stream))
    assert np.array_equal(out[:int(cnt.item())].cpu().numpy().astype(np.int64), want)


@pytest.mark.gpu
def test_gpu_exact_counts_at_every_capacity():
    import torch
    keys = [b"a", b"ab", b"ba", b"aaa", b"aa", b"aaaaa"]
    A, _ = automaton("bytes", False, [list(k) for k in keys])
    hays = [b"aaaaaaaabaaab" * 30, b"", b"ba" * 40, b"c"]
    want = rows(A.find_leftmost_first_batch(hays))
    n = len(want)
    assert n > 10
    L = N.lib()
    tb, flat, offs = table_and_batch(A, hays)
    check_host_capacities(lambda out, cap, found: L.acb_scan_host_leftmost_kind(
        tb, N.SELECT_FIRST, N.ptr(flat), flat.size, N.ptr(offs), len(hays), 0, None, -1, out, cap, found, N.ALGO_AUTO), want)
    bits, n_bits = _word_bits(("bytes", b"ab"), 1)
    hays_w = hays + [b"a aa ab ba aaa aaaaa " * 10]
    want_w = rows(A.find_leftmost_first_batch(hays_w, whole_words=b"ab"))
    assert len(want_w) > 10
    _, flat_w, offs_w = table_and_batch(A, hays_w)
    check_host_capacities(lambda out, cap, found: L.acb_scan_host_leftmost_kind(
        tb, N.SELECT_FIRST, N.ptr(flat_w), flat_w.size, N.ptr(offs_w), len(hays_w), 0, N.ptr(bits), n_bits, out, cap, found,
        N.ALGO_AUTO), want_w)
    full = A.find_all_batch(hays)
    rec = np.stack([full.hay_id, full.end_index, full.key_id], axis=1).astype(np.int32)
    rec = rec[np.random.default_rng(0).permutation(len(rec))]
    d_rec = torch.from_numpy(np.ascontiguousarray(rec)).cuda()
    check_device_capacities(lambda out, cap, cnt, s: L.acb_leftmost_first_device(
        tb, d_rec.data_ptr(), len(rec), len(hays), int(flat.size), out, cap, cnt, s), want, d_rec)


@pytest.mark.gpu
@pytest.mark.parametrize("fl", ["bytes", "unicode"])
def test_gpu_cuda_tensors_on_a_side_stream(fl):
    import torch
    rng = np.random.default_rng(5)
    case = "bytes" if fl == "bytes" else "wide"
    keys = [list(k) for k in {tuple(rng.choice(CASES[case][2][:2], size=int(rng.integers(1, 6)))) for _ in range(12)}]
    rng.shuffle(keys)
    A, O = automaton(*CASES[case][:2], keys)
    L = A._L
    hays = [[int(x) for x in rng.choice(CASES[case][2], size=7)] for _ in range(300)]
    host = np.stack([np.asarray(h, dtype=DT[L]).view(np.uint8) for h in hays])
    d = torch.from_numpy(host).cuda()
    assert got_values(A.find_leftmost_first_batch(host)) == first_cases.find(case, keys, hays)
    views = {"whole": (d, hays)}
    if L == 1:
        views["misaligned"] = (d[1:], hays[1:])
        assert d[1:].data_ptr() % 16 != 0
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    reps = replace_reps(case, keys, rng)
    R = A.replacer({obj(*CASES[case][:2], k): obj(*CASES[case][:2], r) for k, r in zip(keys, reps)}, leftmost_first=True)
    for name, (t, hs) in views.items():
        with torch.cuda.stream(side):
            m = A.find_leftmost_first_batch(t)
            out, offs = R.replace_batch(t)
        assert got_values(m) == first_cases.find(case, keys, hs), name
        torch.cuda.synchronize()
        assert split(out.cpu().numpy(), offs.cpu().numpy(), L) == first_cases.sub(case, keys, reps, hs), name


@pytest.mark.gpu
def test_gpu_first_and_longest_interleaved_on_one_table():
    """both selections share the table's scratch: calls of either kind on two CUDA streams, none waiting for the host,
    each still gets its own answer"""
    import torch
    from pyahocorasick_b200 import synth
    w = synth.make("C2", scale=0.02)
    keys = list(w.keys)
    np.random.default_rng(2).shuffle(keys)
    A = synth.build_automaton(keys)
    d = torch.from_numpy(w.haystacks).cuda()
    want_first = rows(A.find_leftmost_first_batch(w.haystacks))
    want_longest = rows(A.find_leftmost_longest_batch(w.haystacks))
    assert not np.array_equal(want_first, want_longest)
    tb = A._ensure_table(0)
    full = A.find_all_batch(w.haystacks)
    rec = torch.from_numpy(np.stack([full.hay_id, full.end_index, full.key_id], axis=1).astype(np.int32)).cuda()
    n, n_hay, letters = len(full), w.n_hay, w.haystacks.shape[1]
    L = N.lib()
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    outs = []
    torch.cuda.synchronize()
    for i in range(6):
        s = streams[i % 2]
        out = torch.empty((n, 3), dtype=torch.int32, device="cuda")
        cnt = torch.zeros(1, dtype=torch.int64, device="cuda")
        with torch.cuda.stream(s):
            cnt.zero_()
            fn = L.acb_leftmost_first_device if i % 3 != 1 else L.acb_leftmost_longest_device
            N.check(fn(tb, rec.data_ptr(), n, n_hay, letters, out.data_ptr(), n, cnt.data_ptr(), s.cuda_stream))
        outs.append((i % 3 != 1, out, cnt))
    torch.cuda.synchronize()
    for first, out, cnt in outs:
        got = out[:int(cnt.item())].cpu().numpy().astype(np.int64)
        assert np.array_equal(got, want_first if first else want_longest)
    assert np.array_equal(rows(A.find_leftmost_first_batch(d)), want_first)


# launches of the new host routes: the same as the leftmost-longest routes they mirror (tests/test_host_route_launches.py)
SELECTION = 1 + 1 + 1 + 1 + 2                 # sort key, candidates, successors, chain, emit + count
REPLACEMENT = 3 + 2                           # delta, records, offsets, tiles, write
WORD_FILTER = 1 + 2                           # flags, emit + count
FEED_LEFTMOST = 1 + 2 + 1 + 1 + 1 + 1         # staged lengths, gather tiles + gather, scan, frontier flags, last chosen, frontier
KEYS = [b"he", b"she", b"his", b"hers"]
HAYS = [b"ushers and she sells his shells", b"his hers", b"", b"hehe she said"]


@pytest.mark.gpu
@pytest.mark.parametrize("route", ["scan", "scan_words", "replace", "replace_words", "feed", "feed_words", "streams_replace"])
def test_gpu_launch_counts(route):
    A = pkg.flavour("bytes").Automaton()
    for i, k in enumerate(KEYS):
        A.add_word(k, i)
    A.make_automaton()
    L = N.lib()
    tb, flat, off = table_and_batch(A, HAYS)
    bits, n_bits = _word_bits(("bytes", None), 1)
    words = route.endswith("words")
    wb = (N.ptr(bits), n_bits) if words else (None, -1)
    out = np.empty((1024, 3), dtype=np.int32)
    found = ctypes.c_int64()
    rep = np.frombuffer(b"".join(k.upper() + b"!" for k in KEYS), dtype=np.uint8).copy()
    rep_off = np.cumsum([0] + [len(k) + 1 for k in KEYS]).astype(np.int64)
    out_off = np.empty(len(HAYS) + 1, dtype=np.int64)
    out_b = np.empty(4096, dtype=np.uint8)
    total = ctypes.c_int64()
    batch = (N.ptr(flat), flat.size, N.ptr(off), len(HAYS), 0)

    def run():
        r, ss = ctypes.c_void_p(), ctypes.c_void_p()
        N.check(L.acb_replacer_new_kind(tb, N.SELECT_FIRST, N.ptr(rep), rep.size, N.ptr(rep_off), len(KEYS), ctypes.byref(r)))
        N.check(L.acb_streams_new_leftmost_kind(tb, len(HAYS), N.SELECT_FIRST, *wb, ctypes.byref(ss)))
        try:
            before = L.acb_launch_count()
            if route.startswith("scan"):
                N.check(L.acb_scan_host_leftmost_kind(tb, N.SELECT_FIRST, *batch, *wb, N.ptr(out), 1024, ctypes.byref(found),
                                                      N.ALGO_FILTER))
            elif route == "replace":
                N.check(L.acb_replace_host(r, tb, *batch, N.ALGO_FILTER, N.ptr(out_off), N.ptr(out_b), out_b.size, ctypes.byref(total)))
            elif route == "replace_words":
                N.check(L.acb_replace_host_words(r, tb, *batch, *wb, N.ALGO_FILTER, N.ptr(out_off), N.ptr(out_b), out_b.size,
                                                 ctypes.byref(total)))
            elif route.startswith("feed"):
                N.check(L.acb_streams_feed_leftmost_host(ss, tb, *batch, None, 1, N.ptr(out), 1024, ctypes.byref(found), N.ALGO_FILTER))
            else:
                N.check(L.acb_streams_replace_host(ss, r, tb, *batch, None, 1, N.ALGO_FILTER, N.ptr(out_off), N.ptr(out_b),
                                                   out_b.size, ctypes.byref(total)))
            return L.acb_launch_count() - before
        finally:
            L.acb_streams_free(ss)
            L.acb_replacer_free(r)

    want = {"scan": 1 + SELECTION, "scan_words": 1 + WORD_FILTER + SELECTION, "replace": 1 + SELECTION + REPLACEMENT,
            "replace_words": 1 + WORD_FILTER + SELECTION + REPLACEMENT, "feed": FEED_LEFTMOST + SELECTION + 1,
            "feed_words": FEED_LEFTMOST + SELECTION + 1 + 1, "streams_replace": FEED_LEFTMOST + SELECTION + 2 + REPLACEMENT + 1}
    run()                                                      # first call: every workspace is grown
    assert run() == want[route]


@pytest.mark.gpu
def test_gpu_replacing_feed_refuses_a_replacer_of_the_other_kind():
    A = pkg.flavour("bytes").Automaton()
    for i, k in enumerate(KEYS):
        A.add_word(k, i)
    A.make_automaton()
    L = N.lib()
    tb, flat, off = table_and_batch(A, HAYS)
    rep = np.frombuffer(b"".join(KEYS), dtype=np.uint8).copy()
    rep_off = np.cumsum([0] + [len(k) for k in KEYS]).astype(np.int64)
    out_off = np.empty(len(HAYS) + 1, dtype=np.int64)
    out_b = np.empty(4096, dtype=np.uint8)
    total = ctypes.c_int64()
    for batch_kind, rep_kind in ((N.SELECT_FIRST, N.SELECT_LONGEST), (N.SELECT_LONGEST, N.SELECT_FIRST)):
        r, ss = ctypes.c_void_p(), ctypes.c_void_p()
        N.check(L.acb_replacer_new_kind(tb, rep_kind, N.ptr(rep), rep.size, N.ptr(rep_off), len(KEYS), ctypes.byref(r)))
        N.check(L.acb_streams_new_leftmost_kind(tb, len(HAYS), batch_kind, None, -1, ctypes.byref(ss)))
        try:
            assert L.acb_streams_replace_host(ss, r, tb, N.ptr(flat), flat.size, N.ptr(off), len(HAYS), 0, None, 1, N.ALGO_FILTER,
                                              N.ptr(out_off), N.ptr(out_b), out_b.size, ctypes.byref(total)) == N.ACB_EINVAL
        finally:
            L.acb_streams_free(ss)
            L.acb_replacer_free(r)
