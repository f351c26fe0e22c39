"""Automaton.stream_batch(): the next chunk of many streams in one call.

Every randomised test has a CPU form, which runs the Python layer on the emulated feed (tests/emul_streams.py), and a
gpu-marked twin with its own seeds on the real kernels.  The answer for stream s is always the C oracle's (or the
drop-in's already pinned iter_long().set() chain) over the concatenation of s's chunks: a feed must report exactly
the records that end inside its chunks, at their positions in the streams, in the reference's order."""
import ctypes

import numpy as np
import pytest

import emul
import emul_streams
import pyahocorasick_b200 as pkg
from batch_cases import automaton, got_values, obj, triples
from pyahocorasick_b200 import _native as N

# (flavour, key type): 1-, 2- and 4-byte letters
KINDS = {"bytes": ("bytes", False), "seq": ("bytes", True), "unicode": ("unicode", False)}


ALPHA = {"bytes": [0x61, 0x62, 0x63], "seq": [0x61, 0x6162, 0xFFFF], "unicode": [0x61, 0x142, 0x1F600]}


def _keys(kind, rng, lo=1, hi=20, n=12):
    al = ALPHA[kind]
    keys = {tuple(int(x) for x in rng.choice(al, size=int(rng.integers(lo, hi + 1)))) for _ in range(n)}
    return sorted(keys)


def _chunk(kind, rng, T):
    """empty, one letter, shorter than T (a key then straddles three chunks or more), or longer"""
    r = int(rng.integers(0, 6))
    n = [0, 1, max(T - 1, 0), int(rng.integers(0, max(T, 1) + 1)), int(rng.integers(T, 3 * T + 8)), 40][r]
    return [int(x) for x in rng.choice(ALPHA[kind], size=n)]


def _run(A, O, kind, rng, n_streams, n_feeds, algo="auto"):
    """feed random chunks to random subsets of streams; compare every feed with the oracle over the concatenations"""
    S = A.stream_batch(n_streams, algo=algo)
    T = A.get_stats()["longest_word"] - 1
    hist = [[] for _ in range(n_streams)]
    for _ in range(n_feeds):
        if rng.integers(0, 2):
            ids = rng.permutation(n_streams)[:int(rng.integers(0, n_streams + 1))]
        else:
            ids = None
        sel = list(range(n_streams)) if ids is None else ids.tolist()
        chunks = [_chunk(kind, rng, T) for _ in sel]
        m = S.feed([obj(*KINDS[kind], c) if c or rng.integers(0, 2) else None for c in chunks], ids)
        want = []
        for s, c in zip(sel, chunks):
            before = len(hist[s])
            hist[s] += c
            for e, v in O.find_all(obj(*KINDS[kind], hist[s])) or []:
                if e >= before:
                    want.append((s, e, v))
        got = triples(m)
        assert got == want
        assert S.positions.tolist() == [len(h) for h in hist]
    return S, hist


# ------------------------------------------------------------------ differential against the C oracle
def _differential(kind, seed, n_streams, trials, algo="auto"):
    rng = np.random.default_rng(seed)
    for t in range(trials):
        hi = 1 if t == 0 else 20                                # T = 0 once
        A, O = automaton(*KINDS[kind], _keys(kind, rng, hi=hi))
        _run(A, O, kind, rng, n_streams, 6, algo=algo)


@pytest.mark.parametrize("algo", ["filter", "dfa"])
@pytest.mark.parametrize("kind", list(KINDS))
def test_streams_match_oracle_emulated(kind, algo, monkeypatch):
    emul_streams.install(monkeypatch, algo)
    _differential(kind, 11, 12, 3, algo)


@pytest.mark.gpu
@pytest.mark.parametrize("algo", ["filter", "dfa"])
@pytest.mark.parametrize("kind", list(KINDS))
def test_streams_match_oracle_gpu(kind, algo):
    _differential(kind, 1011, 300, 4, algo)


# forced filter shapes: the pair placement, a single-placement stream shape, the tag bitmap
SHAPES = [("bytes", "4,1,0,1", False), ("bytes", "3,2,0,0", False), ("bytes", "4,1,0,1", True), ("unicode", "8,4,0,0", True)]


@pytest.mark.gpu
@pytest.mark.parametrize("kind,env,tagmap", SHAPES)
def test_streams_on_forced_filter_shapes_gpu(kind, env, tagmap, monkeypatch):
    rng = np.random.default_rng(2024)
    g, s = int(env.split(",")[0]), int(env.split(",")[1])
    L = 4 if kind == "unicode" else 1
    m = (g + s - L) // L                                        # the shortest key: the forced gram is the longest it allows
    keys = _keys(kind, rng, lo=m, hi=20) + [tuple([ALPHA[kind][1]] * m)]
    A, O = automaton(*KINDS[kind], sorted(set(keys)), monkeypatch, env, tagmap)
    fs = A.filter_shape()
    assert (fs["gram_bytes"], fs["stride"]) == (g, s) and bool(fs["filter_flags"] & emul.FILTER_PAIR) == env.endswith(",1")
    assert bool(fs["log2_bits3"]) == tagmap
    _run(A, O, kind, rng, 200, 6, algo="filter")


def test_streams_equal_iter_set_chain_emulated(monkeypatch):
    """long=False is the reference's iter(c0) run to exhaustion, then set(c1), ... (the C oracle's iterator)"""
    emul_streams.install(monkeypatch)
    rng = np.random.default_rng(5)
    A, O = automaton("bytes", False, _keys("bytes", rng, hi=7))
    S = A.stream_batch(3)
    its, got, want = [None] * 3, [[] for _ in range(3)], [[] for _ in range(3)]
    for _ in range(8):
        chunks = [bytes(rng.choice(ALPHA["bytes"], size=int(rng.integers(0, 9))).tolist()) for _ in range(3)]
        m = S.feed(chunks)
        for s, e, v in zip(m.hay_id.tolist(), m.end_index.tolist(), m.values()):
            got[s].append((e, v))
        for s in range(3):
            if its[s] is None:
                its[s] = O.iter(chunks[s])
            else:
                its[s].set(chunks[s])
            want[s] += list(its[s])
    assert got == want


# ------------------------------------------------------------------ planted seams
def _planted(seed, residues, n_keys_extra):
    """a key cut at every split point across a feed boundary, behind every residue of the filter stride"""
    rng = np.random.default_rng(seed)
    key = b"qrstuvwxyzQR"
    keys = [tuple(key)] + [tuple(rng.integers(0x61, 0x65, size=int(rng.integers(5, 13))).tolist()) for _ in range(n_keys_extra)]
    A, O = automaton("bytes", False, keys)
    cases = [(r, j) for r in range(residues) for j in range(1, len(key))]
    S = A.stream_batch(len(cases))
    m0 = S.feed([b"0" * r + key[:j] for r, j in cases])
    m1 = S.feed([key[j:] + b"0" * 5 for r, j in cases])
    assert len(m0) == 0
    assert m1.hay_id.tolist() == list(range(len(cases)))
    assert m1.end_index.tolist() == [r + len(key) - 1 for r, j in cases]
    assert m1.key_id.tolist() == [0] * len(cases)


def test_planted_seams_emulated(monkeypatch):
    emul_streams.install(monkeypatch)
    _planted(3, 4, 3)


@pytest.mark.gpu
def test_planted_seams_gpu():
    _planted(1003, 16, 40)


# ------------------------------------------------------------------ iter_long streams
def _long_chain(kind, seed, n_streams, trials):
    """long=True: stream s equals the drop-in's own iter_long(c0) -> exhaust -> set(c1) chain"""
    rng = np.random.default_rng(seed)
    for _ in range(trials):
        A, O = automaton(*KINDS[kind], _keys(kind, rng, hi=8))
        S = A.stream_batch(n_streams, long=True)
        its = [None] * n_streams
        for _ in range(6):
            ids = rng.permutation(n_streams)[:int(rng.integers(1, n_streams + 1))]
            chunks = [obj(*KINDS[kind], _chunk(kind, rng, 6)) for _ in ids]
            m = S.feed(chunks, ids)
            want = []
            for s, c in zip(ids.tolist(), chunks):
                if its[s] is None:
                    its[s] = A.iter_long(c)
                else:
                    its[s].set(c)
                want += [(s, e, v) for e, v in its[s]]
            assert got_values(m) == want


@pytest.mark.parametrize("kind", list(KINDS))
def test_long_streams_equal_iter_long_set_emulated(kind, monkeypatch):
    emul.install(monkeypatch)
    emul_streams.install(monkeypatch)
    _long_chain(kind, 21, 6, 3)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", list(KINDS))
def test_long_streams_equal_iter_long_set_gpu(kind):
    _long_chain(kind, 1021, 64, 3)


# ------------------------------------------------------------------ reset, key-set changes, independence
def _reset_and_independence():
    rng = np.random.default_rng(8)
    A, O = automaton("bytes", False, _keys("bytes", rng, hi=6))
    S1, S2 = A.stream_batch(4), A.stream_batch(4)
    S1.feed([b"abcab", b"ca", b"", b"bbb"])
    S1.reset([1, 3])
    fresh = A.stream_batch(4)
    x = [b"cabcab", b"abcabc", b"a", b"cc"]
    a, b = S1.feed(x), fresh.feed(x)
    for s in (1, 3):
        assert [(e, k) for h, e, k in zip(a.hay_id, a.end_index, a.key_id) if h == s] == \
               [(e, k) for h, e, k in zip(b.hay_id, b.end_index, b.key_id) if h == s]
    assert S1.positions.tolist() == [11, 6, 1, 2]
    assert S2.positions.tolist() == [0, 0, 0, 0]                 # an independent batch did not move
    S1.reset()
    assert S1.positions.tolist() == [0, 0, 0, 0]
    A.add_word(b"zz", 99)
    A.make_automaton()
    for call in (lambda: S1.feed([b"a"]), lambda: S1.reset(), lambda: S2.feed([b"a"], [0])):
        with pytest.raises(ValueError, match="underlaying automaton has changed"):
            call()


def test_reset_independence_and_key_set_change_emulated(monkeypatch):
    emul_streams.install(monkeypatch)
    _reset_and_independence()


@pytest.mark.gpu
def test_reset_independence_and_key_set_change_gpu():
    _reset_and_independence()


def test_argument_errors(monkeypatch):
    emul_streams.install(monkeypatch)
    A, _ = automaton("bytes", False, [tuple(b"ab")])
    S = A.stream_batch(3)
    with pytest.raises(ValueError):
        S.feed([b"a", b"b"], [1, 1])                            # duplicate
    with pytest.raises(ValueError):
        S.feed([b"a"], [3])                                     # out of range
    with pytest.raises(ValueError):
        S.feed([b"a"], [-1])
    with pytest.raises(ValueError):
        S.feed([b"a"] * 4)                                      # more chunks than streams, no ids
    with pytest.raises(ValueError):
        S.feed([b"a", b"b"], [0])                               # one id per chunk
    assert S.positions.tolist() == [0, 0, 0]                    # nothing ran
    U, _ = automaton("unicode", False, [tuple(b"ab")])
    with pytest.raises(ValueError, match="multiple of the letter width"):
        U.stream_batch(2).feed(np.zeros((2, 6), dtype=np.uint8))
    E = pkg.flavour("bytes").Automaton()
    with pytest.raises(AttributeError):
        E.stream_batch(2)
    with pytest.raises(ValueError):
        A.stream_batch(2, algo="long")
    with pytest.raises(ValueError):
        A.stream_batch(2, long=True, algo="dfa")


# ------------------------------------------------------------------ GPU only: the C ABI, overflow, device input
def _c(A):
    return A._lib, A._ensure_table(0)


@pytest.mark.gpu
def test_c_abi_refuses_a_table_of_another_key_set():
    A, _ = automaton("bytes", False, [tuple(b"abc")])
    B, _ = automaton("bytes", False, [tuple(b"abcdef")])
    U, _ = automaton("unicode", False, [tuple(b"abc")])
    lib, ta = _c(A)
    ss = ctypes.c_void_p()
    N.check(lib.acb_streams_new(ta, 4, 0, ctypes.byref(ss)))
    try:
        buf = np.frombuffer(b"abcabc", dtype=np.uint8).copy()
        n = ctypes.c_int64(0)
        for other in (B, U):                                      # another tail length, another letter width
            assert lib.acb_streams_feed_host(ss, other._ensure_table(0), N.ptr(buf), 6, None, 1, 6, None, None, 64,
                                             ctypes.byref(n), 0, 1) == N.ACB_EINVAL
        ids = np.array([2, 2], dtype=np.int32)
        assert lib.acb_streams_feed_host(ss, ta, N.ptr(buf), 6, None, 2, 3, N.ptr(ids), None, 64, ctypes.byref(n), 0, 1) == N.ACB_EINVAL
        assert lib.acb_streams_feed_host(ss, ta, N.ptr(buf), 6, None, 6, 1, None, None, 64, ctypes.byref(n), 0, 1) == N.ACB_EINVAL
        pos = np.zeros(4, dtype=np.int64)
        N.check(lib.acb_streams_positions(ss, N.ptr(pos), 4))
        assert pos.tolist() == [0, 0, 0, 0]
    finally:
        lib.acb_streams_free(ss)


def _overflow(device_route, long_mode=0):
    """caps 0, 1, n-1, n, n+1 with records of keys that began in the chunk before (long_mode: streams that enter the
    feed inside a key, in a non-root state): exact count, no stream advanced; the retry gives what a twin batch fed with
    room gives, and so does every later feed"""
    import torch
    rng = np.random.default_rng(77)
    key_len = np.array([2, 2, 3, 1])
    A, _ = automaton("bytes", False, [tuple(b"ab"), tuple(b"ba"), tuple(b"aba"), tuple(b"b")])
    lib, tb = _c(A)
    n_streams, stride = 64, 32
    feeds = [rng.choice(np.frombuffer(b"ab", dtype=np.uint8), size=(n_streams, stride)) for _ in range(3)]
    twin, ss = ctypes.c_void_p(), ctypes.c_void_p()
    N.check(lib.acb_streams_new(tb, n_streams, long_mode, ctypes.byref(twin)))
    N.check(lib.acb_streams_new(tb, n_streams, long_mode, ctypes.byref(ss)))

    def feed(h, batch, cap):
        if device_route:
            d = torch.from_numpy(batch).cuda()
            out = torch.zeros((max(cap, 1), 3), dtype=torch.int32, device="cuda")
            cnt = torch.full((1,), 12345, dtype=torch.int64, device="cuda")
            N.check(lib.acb_streams_feed_device(h, tb, d.data_ptr(), batch.size, None, n_streams, stride, None,
                                                out.data_ptr(), cap, cnt.data_ptr(), torch.cuda.current_stream().cuda_stream, 0))
            n = int(cnt.item())
            if n > cap:
                return n, None
            N.check(lib.acb_sort_matches_device(tb, out.data_ptr(), n, n_streams, stride, torch.cuda.current_stream().cuda_stream))
            return n, out[:n].cpu().numpy().copy()
        out = np.zeros((max(cap, 1), 3), dtype=np.int32)
        n = ctypes.c_int64(0)
        rc = lib.acb_streams_feed_host(h, tb, N.ptr(batch), batch.size, None, n_streams, stride, None, N.ptr(out), cap,
                                       ctypes.byref(n), 0, 1)
        if rc == N.ACB_EOVERFLOW:
            return n.value, None
        N.check(rc)
        return n.value, out[:n.value].copy()

    def positions(h):
        p = np.zeros(n_streams, dtype=np.int64)
        N.check(lib.acb_streams_positions(h, N.ptr(p), n_streams))
        return p.tolist()

    try:
        for k, batch in enumerate(feeds):
            n, want = feed(twin, batch, 1 << 16)
            if k:                                               # records of keys that began in the chunk before
                assert np.any(want[:, 1] - key_len[want[:, 2]] + 1 < 0)
            for cap in (0, 1, n - 1):
                got_n, got = feed(ss, batch, cap)
                assert (got_n, got) == (n, None)
                assert positions(ss) == [stride * k] * n_streams
            got_n, got = feed(ss, batch, n + (k & 1))           # the retry, with room: n, then n + 1
            assert got_n == n and np.array_equal(got, want)
            assert positions(ss) == positions(twin) == [stride * (k + 1)] * n_streams
    finally:
        lib.acb_streams_free(ss)
        lib.acb_streams_free(twin)


@pytest.mark.gpu
def test_overflow_commits_nothing_host_gpu():
    _overflow(False)


@pytest.mark.gpu
def test_overflow_commits_nothing_device_gpu():
    _overflow(True)


@pytest.mark.gpu
def test_overflow_commits_nothing_long_host_gpu():
    _overflow(False, long_mode=1)


@pytest.mark.gpu
def test_overflow_commits_nothing_long_device_gpu():
    _overflow(True, long_mode=1)


@pytest.mark.gpu
def test_device_tensor_feed_equals_host_feed():
    import torch
    rng = np.random.default_rng(31)
    A, _ = automaton("bytes", False, _keys("bytes", rng, hi=12))
    Sh, Sd = A.stream_batch(500), A.stream_batch(500)
    for k in range(4):
        batch = rng.choice(np.frombuffer(b"abc", dtype=np.uint8), size=(300, 7 + k))
        ids = rng.permutation(500)[:300]
        mh = Sh.feed(batch, ids)
        md = Sd.feed(torch.from_numpy(batch).cuda(), ids)
        for a in ("hay_id", "end_index", "key_id"):
            assert getattr(mh, a).tolist() == getattr(md, a).tolist()
        assert Sh.positions.tolist() == Sd.positions.tolist()


@pytest.mark.gpu
def test_position_past_2_31_is_exact():
    """one stream, three 1 GiB device chunks, a key across 2^31"""
    import torch
    A, _ = automaton("bytes", False, [tuple(b"abcd")])
    S = A.stream_batch(1)
    G = 1 << 30
    d = torch.zeros((1, G), dtype=torch.uint8, device="cuda")
    assert len(S.feed(d)) == 0
    d[0, -2:] = torch.tensor(list(b"ab"), dtype=torch.uint8)
    assert len(S.feed(d)) == 0
    d[0, -2:] = 0
    d[0, :2] = torch.tensor(list(b"cd"), dtype=torch.uint8)
    m = S.feed(d)
    del d
    assert m.hay_id.tolist() == [0] and m.end_index.tolist() == [2 ** 31 + 1] and m.end_index.dtype == np.int64
    assert S.positions.tolist() == [3 * G]
