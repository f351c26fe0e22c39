"""find_leftmost_longest_batch / acb_leftmost_longest_device / acb_scan_host_leftmost: leftmost-longest non-overlapping
matches selected on the GPU from the full match list.

The answer is always the definition (emul_leftmost.greedy) over the full list of the C oracle (per-haystack iter()), or,
at scale, over the full list find_all_batch returns for the same batch.  The CPU tests run the numpy restatement of the
device steps (tests/emul_leftmost.py) at tiny tile sizes; the gpu-marked tests run the real kernels."""
import ctypes

import numpy as np
import pytest

import emul_leftmost
import oracle
import pyahocorasick_b200 as pkg
from batch_cases import (CASES, DT, automaton, check_device_capacities, check_host_capacities, fake_table, forms,
                         got_values, key_len, leftmost_random_case, leftmost_structured_cases, np_greedy, obj, oracle_full,
                         rows, skip_if_device, table_and_batch)
from pyahocorasick_b200 import _native as N

TILES = [1, 2, 3, 7]


def _want(O, keys, hays, case="bytes"):
    return emul_leftmost.greedy(oracle_full(O, hays, case), [len(k) for k in keys])


# ------------------------------------------------------------------ the restatement against the definition (CPU)
@pytest.mark.parametrize("tile", TILES + [2048])
def test_restatement_equals_the_definition_on_the_oracle(tile):
    rng = np.random.default_rng(tile)
    for case, (fl, seq, _) in CASES.items():
        for _ in range(12):
            keys, hays = leftmost_random_case(case, rng)
            _, O = automaton(fl, seq, keys)
            full = oracle_full(O, hays, case)
            kl = np.array([len(k) for k in keys])
            raw = np.array(full, dtype=np.int64).reshape(-1, 3)
            got = emul_leftmost.select(raw[rng.permutation(len(raw))], kl, int(kl.max()), tile)
            assert [tuple(r) for r in got.tolist()] == emul_leftmost.greedy(full, kl), (case, keys, hays)
    for keys, hays in leftmost_structured_cases():
        _, O = automaton("bytes", False, keys)
        full = oracle_full(O, hays)
        kl = np.array([len(k) for k in keys])
        got = emul_leftmost.select(np.array(full, dtype=np.int64).reshape(-1, 3), kl, int(kl.max()), tile)
        assert [tuple(r) for r in got.tolist()] == emul_leftmost.greedy(full, kl)


@pytest.mark.parametrize("tile", TILES)
def test_chains_enter_tiles_at_every_offset(tile):
    """one haystack of runs of a under keys a^1 .. a^W: next(i) = i + W inside a run, so W chains never meet and
    every tile depends on its entry; the runs' lengths move the entry across every offset"""
    rng = np.random.default_rng(100 + tile)
    for W in (1, 2, 5, 16):
        keys = [[0x61] * k for k in range(1, W + 1)]
        _, O = automaton("bytes", False, keys)
        hay = []
        for _ in range(30):
            hay += [0x61] * int(rng.integers(1, 3 * W + 2)) + [0x62]
        full = oracle_full(O, [hay, hay[:17], hay])
        kl = np.array([len(k) for k in keys])
        got = emul_leftmost.select(np.array(full, dtype=np.int64).reshape(-1, 3), kl, W, tile)
        assert [tuple(r) for r in got.tolist()] == emul_leftmost.greedy(full, kl)


@pytest.mark.parametrize("tile", [1, 3, 2048])
def test_python_layer_on_the_restatement(monkeypatch, tile):
    emul_leftmost.install(monkeypatch, tile)
    rng = np.random.default_rng(7 + tile)
    for case, (fl, seq, _) in CASES.items():
        for _ in range(4):
            keys, hays = leftmost_random_case(case, rng)
            A, O = automaton(fl, seq, keys)
            want = _want(O, keys, hays, case)
            for form, batch in forms([obj(fl, seq, h) for h in hays], hays, A._L, case in ("latin1", "mixed")):
                assert got_values(A.find_leftmost_longest_batch(batch)) == want, (case, form)
    for keys, hays in leftmost_structured_cases():
        A, O = automaton("bytes", False, keys)
        assert got_values(A.find_leftmost_longest_batch([bytes(h) for h in hays])) == _want(O, keys, hays)


def test_abcde_example_differs_from_iter_long(monkeypatch):
    """keys abcde, bcdx, cd and the text abcdy: iter_long reports nothing (its restart rule checks only a node and its
    direct fail link), iter reports (3, cd), and leftmost-longest takes cd"""
    emul_leftmost.install(monkeypatch)
    keys = [b"abcde", b"bcdx", b"cd"]
    A, O = automaton("bytes", False, keys)
    assert list(O.iter_long(b"abcdy")) == []
    assert list(O.iter(b"abcdy")) == [(3, 2)]
    if oracle.ref_available("bytes"):
        R = oracle.ref_module("bytes").Automaton()
        for i, k in enumerate(keys):
            R.add_word(k, i)
        R.make_automaton()
        assert list(R.iter_long(b"abcdy")) == []
        assert list(R.iter(b"abcdy")) == [(3, 2)]
    assert got_values(A.find_leftmost_longest_batch([b"abcdy"])) == [(0, 3, 2)]


def test_argument_errors():
    mod = pkg.flavour("bytes")
    A = mod.Automaton()
    A.add_word(b"ab", 0)
    with pytest.raises(AttributeError):
        A.find_leftmost_longest_batch([b"ab"])                 # not built: what find_all_batch raises
    with pytest.raises(AttributeError):
        A.find_all_batch([b"ab"])
    A.make_automaton()
    for algo in ("long", "x"):
        with pytest.raises(ValueError):
            A.find_leftmost_longest_batch([b"ab"], algo=algo)
    L = N.lib()
    fake = fake_table()                                         # device 0; never used past the checks
    n = ctypes.c_int64(0)
    hay = np.zeros(16, dtype=np.uint8)
    assert L.acb_scan_host_leftmost(None, N.ptr(hay), 16, None, 1, 16, None, 8, ctypes.byref(n), N.ALGO_AUTO) == N.ACB_EINVAL
    assert L.acb_scan_host_leftmost(ctypes.addressof(fake), N.ptr(hay), 16, None, 1, 16, None, 8, ctypes.byref(n), N.ALGO_LONG) == N.ACB_EINVAL
    assert L.acb_scan_host_leftmost(ctypes.addressof(fake), N.ptr(hay), 16, None, 1, 16, None, -1, ctypes.byref(n), N.ALGO_AUTO) == N.ACB_EINVAL
    cnt = np.zeros(1, dtype=np.int64)
    assert L.acb_leftmost_longest_device(None, N.ptr(hay), 1, 1, 16, N.ptr(hay), 1, N.ptr(cnt), None) == N.ACB_EINVAL
    assert L.acb_leftmost_longest_device(ctypes.addressof(fake), None, 1, 1, 16, N.ptr(hay), 1, N.ptr(cnt), None) == N.ACB_EINVAL
    assert L.acb_leftmost_longest_device(ctypes.addressof(fake), N.ptr(hay), 1, 1, 16, None, 1, N.ptr(cnt), None) == N.ACB_EINVAL
    assert L.acb_leftmost_longest_device(ctypes.addressof(fake), N.ptr(hay), 1 << 31, 1, 16, N.ptr(hay), 1, N.ptr(cnt), None) == N.ACB_ERANGE
    ms = (ctypes.c_float * 5)()
    assert L.acb_last_leftmost_ms(ms, 6) == N.ACB_EINVAL and L.acb_last_leftmost_ms(ms, 5) == N.ACB_OK


def test_host_route_fails_loudly_without_a_device():
    skip_if_device()
    fake = fake_table()
    n = ctypes.c_int64(0)
    hay = np.frombuffer(b"abcd" * 4, dtype=np.uint8)
    offs = np.array([0, 8, 16], dtype=np.int64)
    assert N.lib().acb_scan_host_leftmost(ctypes.addressof(fake), N.ptr(hay), 16, N.ptr(offs), 2, 0, None, 8, ctypes.byref(n), N.ALGO_AUTO) == N.ACB_ECUDA
    assert N.last_error()


# ------------------------------------------------------------------ the real kernels
@pytest.mark.gpu
@pytest.mark.parametrize("algo", ["filter", "dfa"])
def test_gpu_fuzz_against_the_definition(algo):
    rng = np.random.default_rng(11)
    for case, (fl, seq, _) in CASES.items():
        for _ in range(6):
            keys, hays = leftmost_random_case(case, rng)
            A, O = automaton(fl, seq, keys)
            want = _want(O, keys, hays, case)
            for form, batch in forms([obj(fl, seq, h) for h in hays], hays, A._L, case in ("latin1", "mixed")):
                assert got_values(A.find_leftmost_longest_batch(batch, algo=algo)) == want, (case, form, keys, hays)
    for keys, hays in leftmost_structured_cases():
        A, O = automaton("bytes", False, keys)
        assert got_values(A.find_leftmost_longest_batch([bytes(h) for h in hays], algo=algo)) == _want(O, keys, hays)
    A, _ = automaton("bytes", False, [list(b"abcde"), list(b"bcdx"), list(b"cd")])
    assert got_values(A.find_leftmost_longest_batch([b"abcdy"], algo=algo)) == [(0, 3, 2)]
    assert list(A.iter_long(b"abcdy")) == []


@pytest.mark.gpu
def test_gpu_filter_and_dfa_identical_and_ragged():
    from pyahocorasick_b200 import synth
    w = synth.make("C2", scale=0.01)
    A = synth.build_automaton(w.keys)
    rng = np.random.default_rng(3)
    flat = w.haystacks.reshape(-1)
    cuts = rng.integers(0, flat.size, size=3000)
    cuts = np.concatenate([cuts, cuts[:200]])                                   # repeated cuts: empty haystacks
    offs = np.concatenate([[0], np.sort(cuts), [flat.size]]).astype(np.int64)
    for batch in (w.haystacks, (flat, offs)):
        f = A.find_leftmost_longest_batch(batch, algo="filter")
        d = A.find_leftmost_longest_batch(batch, algo="dfa")
        assert np.array_equal(rows(f), rows(d))
        full = A.find_all_batch(batch, algo="filter")
        assert np.array_equal(rows(f), np_greedy(np.rec.fromarrays([full.hay_id, full.end_index, full.key_id],
                                                                    names="hay_id,end_index,key_id"), key_len(A)))
    assert (np.diff(offs) == 0).any()


@pytest.mark.gpu
@pytest.mark.parametrize("fl", ["bytes", "unicode"])
def test_gpu_cuda_tensors_on_a_side_stream(fl):
    import torch
    rng = np.random.default_rng(5)
    case = "bytes" if fl == "bytes" else "wide"
    keys = [list(k) for k in ({tuple(rng.choice(CASES[case][2][:2], size=int(rng.integers(1, 6)))) for _ in range(12)})]
    A, O = automaton(*CASES[case][:2], keys)
    L = A._L
    hays = [[int(x) for x in rng.choice(CASES[case][2], size=7)] for _ in range(300)]
    host = np.stack([np.asarray(h, dtype=DT[L]).view(np.uint8) for h in hays])
    d = torch.from_numpy(host).cuda()
    want = got_values(A.find_leftmost_longest_batch(host))
    assert want == _want(O, keys, hays, case)
    views = {"whole": (d, hays)}
    if L == 1:
        views["misaligned"] = (d[1:], hays[1:])
        assert d[1:].data_ptr() % 16 != 0
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    for name, (t, hs) in views.items():
        with torch.cuda.stream(side):
            m = A.find_leftmost_longest_batch(t)
        assert got_values(m) == _want(O, keys, hs, case), name


@pytest.mark.gpu
def test_gpu_exact_counts_at_every_capacity():
    import torch
    keys = [b"a" * k for k in range(1, 6)] + [b"ab", b"ba"]
    A, _ = automaton("bytes", False, keys)
    hays = [b"aaaaaaaabaaab" * 30, b"", b"ba" * 40, b"c"]
    want = rows(A.find_leftmost_longest_batch(hays))
    n = len(want)
    assert n > 10
    L = N.lib()
    tb, flat, offs = table_and_batch(A, hays)
    check_host_capacities(lambda out, cap, found: L.acb_scan_host_leftmost(
        tb, N.ptr(flat), flat.size, N.ptr(offs), len(hays), 0, out, cap, found, N.ALGO_AUTO), want)
    # the device entry: the full list in any order
    full = A.find_all_batch(hays)
    rec = np.stack([full.hay_id, full.end_index, full.key_id], axis=1).astype(np.int32)
    rec = rec[np.random.default_rng(0).permutation(len(rec))]
    d_rec = torch.from_numpy(np.ascontiguousarray(rec)).cuda()
    check_device_capacities(lambda out, cap, cnt, s: L.acb_leftmost_longest_device(
        tb, d_rec.data_ptr(), len(rec), len(hays), int(flat.size), out, cap, cnt, s), want, d_rec)


@pytest.mark.gpu
def test_gpu_one_haystack_over_many_tiles():
    """runs of a under a^1 .. a^W: W chains that never meet, so every tile depends on its entry (the look-back chain);
    runs of random length move the entry across every offset up to W; plus random text that mixes both regimes"""
    rng = np.random.default_rng(9)
    for W in (1, 3, 16, 64):
        keys = [b"a" * k for k in range(1, W + 1)] + [b"ab", b"ba" * 3]
        A, _ = automaton("bytes", False, keys)
        runs = rng.integers(1, 3 * W + 2, size=40000 // W + 2000)
        hay = b"b".join(b"a" * int(r) for r in runs)
        hays = [hay, b"", hay[: len(hay) // 3], b"ab" * 5000]
        got = A.find_leftmost_longest_batch(hays)
        full = A.find_all_batch(hays)
        want = np_greedy(np.rec.fromarrays([full.hay_id, full.end_index, full.key_id], names="hay_id,end_index,key_id"), key_len(A))
        assert len(want) > 3 * 2048
        assert np.array_equal(rows(got), want), W


def _windows_agree(O, text: bytes, got: np.ndarray, key_len, max_len, rng, n=40, span=1 << 16):
    """from any chosen match the rule restarts exactly: the oracle's matches of a window that starts there, run
    through the definition, agree with the GPU's choices up to a key length before the window's end.  got: (hay, end,
    value) rows; key_len by value"""
    starts = got[:, 1] - key_len[got[:, 2]] + 1
    for i in rng.integers(0, len(got), size=n).tolist():
        s = int(starts[i])
        win = text[s:s + span]
        loc = emul_leftmost.greedy([(0, e, v) for e, v in O.iter(win)], key_len)
        lim = len(win) - max_len
        a = [(e + s, k) for _, e, k in loc if e - key_len[k] + 1 <= lim]
        sel = (starts >= s) & (starts <= s + lim)
        b = list(zip((got[sel, 1]).tolist(), got[sel, 2].tolist()))
        assert a == b


@pytest.mark.gpu
def test_gpu_single_haystack_of_256_mib():
    """one 256 MiB haystack over four letters with keys of 3..6 letters: millions of candidates, checked by a full
    numpy pass of the definition over find_all_batch's list and on sampled windows against the C oracle"""
    rng = np.random.default_rng(21)
    keys = sorted({bytes(rng.choice(list(b"acgt"), size=int(rng.integers(3, 7))).tolist()) for _ in range(24)})
    A, O = automaton("bytes", False, keys)
    text = rng.choice(np.frombuffer(b"acgt", dtype=np.uint8), size=256 << 20)
    offs = np.array([0, text.size], dtype=np.int64)
    m = A.find_leftmost_longest_batch((text, offs))
    got = rows(m)
    full = A.find_all_batch((text, offs))
    kl = key_len(A)
    want = np_greedy(np.rec.fromarrays([full.hay_id, full.end_index, full.key_id], names="hay_id,end_index,key_id"), kl)
    assert len(want) > 2_000_000
    assert np.array_equal(got, want)
    by_value = np.stack([got[:, 0], got[:, 1], np.array(m.values(), dtype=np.int64)], axis=1)
    _windows_agree(O, text.tobytes(), by_value, np.array([len(k) for k in keys]), max(map(len, keys)), rng)


@pytest.mark.gpu
def test_gpu_batch_past_2_gib():
    """a CUDA tensor of 2^31 + 2^24 bytes in 2 080 rows, keys planted near the end of rows and across 2^31"""
    import torch
    keys = [b"qzqzx", b"zqzx", b"qzq", b"xqzqzxq"]
    A, _ = automaton("bytes", False, keys)
    n_rows, stride = 2080, ((1 << 31) + (1 << 24)) // 2080 // 16 * 16
    d = torch.randint(0, 16, (n_rows, stride), dtype=torch.uint8, device="cuda")
    d += ord("a")                                                            # a..p: no key letter but for planted ones
    rng = np.random.default_rng(2)
    for r in rng.integers(0, n_rows, size=400).tolist():
        c = int(rng.integers(0, stride - 8))
        for j, b in enumerate(b"xqzqzxq"[: int(rng.integers(3, 8))]):
            d[r, c + j] = b
    d[-1, -8:] = torch.tensor(list(b"qzqzxqzq"), dtype=torch.uint8)
    got = A.find_leftmost_longest_batch(d)
    full = A.find_all_batch(d)
    want = np_greedy(np.rec.fromarrays([full.hay_id, full.end_index, full.key_id], names="hay_id,end_index,key_id"), key_len(A))
    assert n_rows * stride > (1 << 31) and len(want) > 300
    assert np.array_equal(rows(got), want)


@pytest.mark.gpu
@pytest.mark.parametrize("log_len", [19, 20])
def test_gpu_sort_key_of_64_and_65_bits(log_len):
    """about 128 MiB in 65 536 haystacks and a key of 2^log_len letters that never matches: hay | start | (max_len -
    len) takes 16 + 28 + 20 = 64 bits (one radix sort) or 65 (two stable passes)"""
    rng = np.random.default_rng(log_len)
    short = [b"ab", b"abc", b"bca", b"cab", b"abcab"]
    A, _ = automaton("bytes", False, [list(k) for k in short + [b"d" * (1 << log_len)]])
    n = (128 << 20) + 4096
    text = rng.choice(np.frombuffer(b"abc", dtype=np.uint8), size=n)
    off = np.concatenate([[0], np.sort(rng.integers(0, n, size=65535)), [n]]).astype(np.int64)
    bits = sum(int(v).bit_length() or 1 for v in (len(off) - 2, n, 1 << log_len))
    assert bits == (64 if log_len == 19 else 65)
    got = rows(A.find_leftmost_longest_batch((text, off)))
    full = A.find_all_batch((text, off))
    want = np_greedy(np.rec.fromarrays([full.hay_id, full.end_index, full.key_id], names="hay_id,end_index,key_id"), key_len(A))
    assert np.array_equal(got, want)
