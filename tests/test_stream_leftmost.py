"""stream_batch(leftmost_longest=True) and Replacer.stream_batch: leftmost-longest matches and replacement chunk by chunk.

Whatever the chunking, a stream's feeds plus its finish must give exactly what the whole-batch methods give for its
whole text: emul_leftmost.greedy and emul_replace.definition over the C oracle's full list (CPU and small GPU cases), or
find_leftmost_longest_batch / replace_batch of the whole text on the GPU (at scale).  The CPU tests run the Python layer
on the restatement of the native feed (tests/emul_stream_leftmost.py); the gpu-marked tests run the real kernels."""
import ctypes

import numpy as np
import pytest

import emul_leftmost
import emul_replace
import emul_stream_leftmost
import emul_streams
import pyahocorasick_b200 as pkg
from batch_cases import (CASES, DT, NESTED, automaton, fake_table, leftmost_random_case, obj, oracle_full, replace_reps,
                         rows, skip_if_device, split, table_and_batch)
from pyahocorasick_b200 import _native as N

ABCDE = [[0x61, 0x62, 0x63, 0x64, 0x65], [0x62, 0x63, 0x64, 0x78], [0x63, 0x64]]


def _key_sets(case, rng):
    """random keys, nested keys a .. a^W over runs of a, the abcde / bcdx / cd example, prefixes and suffixes, T = 0"""
    keys, _ = leftmost_random_case(case, rng)
    yield keys
    if case in ("bytes", "latin1", "seq2", "seq4"):
        yield NESTED[:int(rng.integers(2, 9))]
        yield ABCDE
        yield [[0x61, 0x62], [0x61, 0x62, 0x61], [0x62, 0x61], [0x61]]
    yield sorted({(int(x),) for x in rng.choice(CASES[case][2], size=2)})               # T = 0


def _texts(case, keys, rng, n):
    """per stream, a list of segments (texts between finishes)"""
    al = CASES[case][2]
    out = []
    for _ in range(n):
        segs = []
        for _ in range(int(rng.integers(1, 3))):
            r = int(rng.integers(0, 4))
            if r == 0:
                segs.append([])
            elif r == 1:
                segs.append([0x61] * int(rng.integers(1, 60)))
            else:
                body = []
                while len(body) < int(rng.integers(1, 80)):
                    body += list(keys[int(rng.integers(0, len(keys)))]) if rng.integers(0, 2) else \
                        [int(x) for x in rng.choice(al, size=int(rng.integers(1, 4)))]
                segs.append(body)
        out.append(segs)
    return out


def _chunk_len(T, rng):
    return int(rng.choice([0, 1, max(T - 1, 1), max(T, 1), T + 1, 3 * T + 1, int(rng.integers(1, 20))]))


def _drive(case, A, texts, rng, feed, finish, T, check_lag=None):
    """Feed every stream's segments in random chunks: each call takes a random subset of the streams, in random order,
    and an exhausted segment is finished in that call or a later one (empty chunks may come in between).
    feed(chunks, ids) / finish(ids) return per id what it released.  Returns per stream and segment the releases.
    check_lag(stream, segment, position) runs after every feed."""
    n = len(texts)
    seg = [0] * n
    off = [0] * n
    got = [[[] for _ in s] for s in texts]
    while True:
        live = [s for s in range(n) if seg[s] < len(texts[s])]
        if not live:
            return got
        pick = [s for s in rng.permutation(live).tolist() if rng.integers(0, 4)] or live[:1]
        chunks = []
        for s in pick:
            piece = texts[s][seg[s]][off[s]:off[s] + _chunk_len(T, rng)]
            off[s] += len(piece)
            chunks.append(None if not piece and rng.integers(0, 2) else obj(*CASES[case][:2], piece))
        for s, r in zip(pick, feed(chunks, pick)):
            got[s][seg[s]].append(r)
        if check_lag:
            for s in pick:
                check_lag(s, seg[s], off[s])
        done = [s for s in pick if off[s] >= len(texts[s][seg[s]]) and rng.integers(0, 3)]
        if done:
            for s, r in zip(done, finish(done)):
                got[s][seg[s]].append(r)
                seg[s] += 1
                off[s] = 0


def _per_id(m, ids):
    return [[(int(e), int(v)) for h, e, v in zip(m.hay_id.tolist(), m.end_index.tolist(), m.values()) if h == s] for s in ids]


def _want_matches(O, keys, text, case):
    return [(e, k) for _, e, k in emul_leftmost.greedy(oracle_full(O, [text], case), [len(k) for k in keys])]


def _want_output(O, keys, text, reps, case):
    chosen = [(e, k) for _, e, k in emul_leftmost.greedy(oracle_full(O, [text], case), [len(k) for k in keys])]
    return emul_replace.definition(text, chosen, [len(k) for k in keys], reps)


def _letters(case, item):
    if CASES[case][1]:
        return list(item)
    return list(item) if isinstance(item, bytes) else [ord(c) for c in item]


def _run_case(case, keys, texts, rng, algo, emulated):
    fl, seq, _ = CASES[case]
    A, O = automaton(fl, seq, keys)
    T = max(len(k) for k in keys) - 1
    B = A.stream_batch(len(texts), leftmost_longest=True, algo=algo)

    def lag(s, g, p):
        want = _want_matches(O, keys, texts[s][g], case)
        seen = {x for r in got_now[s] for x in r}
        assert {x for x in want if x[0] - len(keys[x[1]]) + 1 < p - T} <= seen, (case, keys, texts[s][g], p)
        if emulated:
            assert len(B._ss["held"][s]) // A._L <= T

    got_now = [[] for _ in texts]

    def feed(chunks, ids):
        r = _per_id(B.feed(chunks, ids), ids)
        for s, x in zip(ids, r):
            got_now[s].append(x)
        return r

    def finish(ids):
        r = _per_id(B.finish(ids), ids)
        for s in ids:
            got_now[s].clear()
        return r

    got = _drive(case, A, texts, rng, feed, finish, T, lag)
    for s, segs in enumerate(texts):
        for g, text in enumerate(segs):
            assert [x for r in got[s][g] for x in r] == _want_matches(O, keys, text, case), (case, algo, keys, text)
    assert not B.positions.any()
    # the replacing form over the same texts
    reps = replace_reps(case, keys, rng)
    R = A.replacer({obj(fl, seq, k): obj(fl, seq, r) for k, r in zip(keys, reps)})
    S = R.stream_batch(len(texts), algo=algo)
    got = _drive(case, A, texts, rng, lambda c, i: [_letters(case, x) for x in S.feed(c, i)],
                 lambda i: [_letters(case, x) for x in S.finish(i)], T)
    for s, segs in enumerate(texts):
        for g, text in enumerate(segs):
            want = _want_output(O, keys, text, reps, case)
            assert [x for r in got[s][g] for x in r] == want, (case, algo, keys, text, reps)
    return A, O, B, S


def _fuzz(algo, emulated, seed, rounds):
    rng = np.random.default_rng(seed)
    for case in CASES:
        for _ in range(rounds):
            for keys in _key_sets(case, rng):
                _run_case(case, [list(k) for k in keys], _texts(case, keys, rng, int(rng.integers(1, 5))), rng, algo, emulated)


# ------------------------------------------------------------------ the Python layer on the restatement (CPU)
def test_python_layer_on_the_restatement(monkeypatch):
    """both flavours, 2- and 4-byte sequences, latin-1 / wide / mixed chunks; nested, prefix, suffix and T = 0 key sets;
    chunks of 1, T-1, T, T+1, 3T+1 letters, empty and None chunks, streams left out of a call, finish mid-stream"""
    emul_stream_leftmost.install(monkeypatch)
    _fuzz("auto", True, 5, 3)


def test_other_input_forms_and_two_interleaved_batches(monkeypatch):
    emul_stream_leftmost.install(monkeypatch)
    emul_replace.install(monkeypatch)
    keys = [b"ab", b"abc", b"bca", b"c"]
    A, O = automaton("bytes", False, keys)
    text = b"abcabcaabcbcab" * 3
    want = [(0, e, k) for e, k in _want_matches(O, [list(k) for k in keys], list(text), "bytes")]
    B1 = A.stream_batch(4, leftmost_longest=True)
    B2 = A.stream_batch(4, leftmost_longest=True)
    got1, got2 = [], []
    for i in range(0, len(text), 6):                      # B1 takes stream 3 as arrays, B2 stream 1 as (flat, offsets)
        piece = np.frombuffer(text[i:i + 6], dtype=np.uint8)
        m = B1.feed(piece[None, :].copy(), ids=[3])
        got1 += list(zip(m.hay_id.tolist(), m.end_index.tolist(), m.values()))
        m = B2.feed((piece, np.array([0, piece.size], np.int64)), ids=[1])
        got2 += list(zip(m.hay_id.tolist(), m.end_index.tolist(), m.values()))
    for B, got, s in ((B1, got1, 3), (B2, got2, 1)):
        assert B.positions[s] == len(text) and B.positions.sum() == len(text)
        m = B.finish([s])
        got += list(zip(m.hay_id.tolist(), m.end_index.tolist(), m.values()))
        assert got == [(s, e, k) for _, e, k in want]
    R = A.replacer({b"ab": b"X", b"abc": b"", b"bca": b"YYYY", b"c": b"c"})
    S = R.stream_batch(2)
    out, offs = S.feed(np.frombuffer(text[:20] + text[:20], dtype=np.uint8).reshape(2, 20))
    assert offs.dtype == np.int64 and len(offs) == 3
    tail = S.finish()
    whole = R.replace_batch([text[:20]])[0]
    assert [out[offs[i]:offs[i + 1]].tobytes() + tail[i] for i in range(2)] == [whole, whole]
    S.feed([b"abc"], ids=[1])
    S.reset([1])
    assert S.finish([1]) == [b""] and not S.positions.any()


def test_argument_errors_and_stale_batches(monkeypatch):
    emul_streams.install(monkeypatch)                     # the find_all batch below
    emul_stream_leftmost.install(monkeypatch)
    mod = pkg.flavour("bytes")
    A = mod.Automaton()
    A.add_word(b"ab", b"X")
    A.make_automaton()
    for kw in ({"long": True}, {"ignore_white_space": True}, {"algo": "long"}):
        with pytest.raises(ValueError):
            A.stream_batch(2, leftmost_longest=True, **kw)
    with pytest.raises(ValueError):
        A.stream_batch(2).finish()                       # finish belongs to leftmost batches
    B = A.stream_batch(2, leftmost_longest=True)
    with pytest.raises(ValueError):
        B.feed([b"a", b"b", b"c"])                       # 3 chunks for 2 streams
    with pytest.raises(ValueError):
        B.feed([b"a", b"b"], ids=[1, 1])
    with pytest.raises(ValueError):
        B.finish([2])
    R = A.replacer()
    with pytest.raises(ValueError):
        R.stream_batch(-1)
    with pytest.raises(ValueError):
        R.stream_batch(1, algo="long")
    S = R.stream_batch(2)
    assert S.feed([b"xa", None]) == [b"x", b""]
    assert S.feed([b"b"]) == [b"X"] and S.finish() == [b"", b""]   # "ab" starts before position 2 - T: settled
    A.add_word(b"cd", b"Y")
    for call in (lambda: B.feed([b"a"]), lambda: B.finish(), lambda: S.feed([b"a"]), lambda: S.finish(),
                 lambda: S.reset(), lambda: R.stream_batch(1)):
        with pytest.raises(ValueError):
            call()


def test_c_entries_check_arguments_first():
    L = N.lib()
    ss = ctypes.c_void_p()
    cnt = np.zeros(4, np.int64)
    hay = np.zeros(32, np.uint8)
    assert L.acb_streams_new_leftmost(None, 1, ctypes.byref(ss)) == N.ACB_EINVAL
    assert L.acb_streams_feed_leftmost_device(None, None, None, 0, None, 0, 0, None, 0, None, 0, N.ptr(cnt), None, 0) == N.ACB_EINVAL
    found = ctypes.c_int64(0)
    assert L.acb_streams_feed_leftmost_host(None, None, N.ptr(hay), 32, None, 1, 32, None, 0, None, 0, ctypes.byref(found), 0) == N.ACB_EINVAL
    assert L.acb_streams_replace_device(None, None, None, N.ptr(hay), 32, None, 1, 32, None, 0, N.ptr(cnt), None, 0, N.ptr(cnt),
                                        None, 0) == N.ACB_EINVAL
    assert L.acb_streams_replace_host(None, None, None, N.ptr(hay), 32, None, 1, 32, None, 0, 0, N.ptr(cnt), None, 0,
                                      ctypes.byref(found)) == N.ACB_EINVAL
    ms = (ctypes.c_float * 6)()
    assert L.acb_last_stream_leftmost_ms(ms, 7) == N.ACB_EINVAL and L.acb_last_stream_leftmost_ms(ms, 6) == N.ACB_OK


def test_c_entries_fail_loudly_without_a_device():
    skip_if_device()
    fake = fake_table(1)
    ss = ctypes.c_void_p()
    assert N.lib().acb_streams_new_leftmost(ctypes.addressof(fake), 4, ctypes.byref(ss)) == N.ACB_ECUDA
    assert N.last_error()


# ------------------------------------------------------------------ the real kernels
@pytest.mark.gpu
@pytest.mark.parametrize("algo", ["filter", "dfa"])
def test_gpu_fuzz_against_the_definition(algo):
    _fuzz(algo, False, 11 if algo == "filter" else 12, 2)


def _rows(text, n):
    return np.frombuffer(text, dtype=np.uint8).reshape(n, -1)


def _collect(B, feeds, n):
    """run B.feed over [(tensor or array, ids)] and finish -> int64 records (stream, end, key id) sorted"""
    recs = []
    for batch, ids in feeds:
        m = B.feed(batch, ids)
        recs.append(np.stack([m.hay_id, m.end_index, m.key_id.astype(np.int64)], axis=1))
    m = B.finish()
    recs.append(np.stack([m.hay_id, m.end_index, m.key_id.astype(np.int64)], axis=1))
    r = np.concatenate(recs)
    return r[np.lexsort((r[:, 1], r[:, 0]))]


def _assemble(outs, n):
    """per-stream concatenation of the feeds' (flat, offsets) outputs, on the host -> (flat, offsets)"""
    lens = np.zeros(n, dtype=np.int64)
    parts = []
    for flat, offs in outs:
        flat, offs = (x.cpu().numpy() if hasattr(x, "cpu") else x for x in (flat, offs))
        parts.append((flat, offs))
        lens += np.diff(offs)
    dst = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(lens, out=dst[1:])
    out = np.empty(int(dst[-1]), dtype=np.uint8)
    cur = dst[:-1].copy()
    for flat, offs in parts:
        ln = np.diff(offs)
        idx = np.repeat(cur - offs[:-1], ln) + np.arange(flat.size)
        out[idx] = flat
        cur += ln
    return out, dst


@pytest.mark.gpu
@pytest.mark.parametrize("step", [256, 1, 7, 64])
def test_gpu_c2_million_streams(step):
    """2^20 streams of the C2 key set (one planted key per 256-byte row) fed `step` letters at a time, so that planted
    keys cross the chunk boundaries, against find_leftmost_longest_batch and replace_batch of the whole rows"""
    import torch
    from pyahocorasick_b200 import synth
    w = synth.make("C2")
    A = synth.build_automaton(w.keys)
    n = w.n_hay
    d = torch.from_numpy(w.haystacks).cuda()
    want = rows(A.find_leftmost_longest_batch(d))
    feeds = [(d[:, i:i + step].contiguous(), None) for i in range(0, d.shape[1], step)]
    got = _collect(A.stream_batch(n, leftmost_longest=True), feeds, n)
    assert np.array_equal(got, want)
    keys = [k for k in A._key_objs if k is not None]
    rng = np.random.default_rng(step)
    table = {k: bytes(rng.integers(0x41, 0x5B, size=int(rng.integers(0, 20)), dtype=np.uint8)) for k in keys}
    R = A.replacer(table)
    wout, woffs = R.replace_batch(d)
    S = R.stream_batch(n)
    outs = [S.feed(t) for t, _ in feeds]
    tail = S.finish()
    flat = np.frombuffer(b"".join(tail), dtype=np.uint8)
    toffs = np.zeros(n + 1, dtype=np.int64)
    np.cumsum([len(x) for x in tail], out=toffs[1:])
    out, offs = _assemble(outs + [(flat, toffs)], n)
    assert np.array_equal(offs, woffs.cpu().numpy()) and np.array_equal(out, wout.cpu().numpy())


@pytest.mark.gpu
@pytest.mark.parametrize("klen", [64, 1000, 5000])
def test_gpu_long_keys(klen):
    rng = np.random.default_rng(klen)
    keys = sorted({bytes(rng.integers(0x61, 0x63, size=int(rng.integers(1, klen + 1)), dtype=np.uint8)) for _ in range(8)}
                  | {bytes(rng.integers(0x61, 0x63, size=klen, dtype=np.uint8))})
    A, _ = automaton("bytes", False, keys)
    n = 6
    texts = []
    for _ in range(n):
        t = b""
        while len(t) < 3 * klen:
            t += keys[int(rng.integers(0, len(keys)))] if rng.integers(0, 2) else bytes(rng.integers(0x61, 0x64, size=5, dtype=np.uint8))
        texts.append(t)
    want = rows(A.find_leftmost_longest_batch(texts))
    R = A.replacer({k: k[: len(k) // 3] for k in keys})
    wout = R.replace_batch(texts)
    B = A.stream_batch(n, leftmost_longest=True)
    S = R.stream_batch(n)
    pos = [0] * n
    feeds, outs = [], [b""] * n
    while any(p < len(t) for p, t in zip(pos, texts)):
        chunks = []
        for s in range(n):
            k = int(rng.choice([1, klen - 2, klen - 1, klen, klen + 1, 3 * klen]))
            chunks.append(texts[s][pos[s]:pos[s] + k])
            pos[s] += k
        feeds.append((chunks, None))
        outs = [a + b for a, b in zip(outs, S.feed(chunks))]
    assert np.array_equal(_collect(B, feeds, n), want)
    assert [a + b for a, b in zip(outs, S.finish())] == wout


@pytest.mark.gpu
def test_gpu_staged_batch_past_2_gib():
    """two chunks of 1.1 GB each: the staged batch passes 2^31 bytes; planted keys cross the feeds' boundary"""
    import torch
    n, size = 2, 1_100_000_000
    d = torch.zeros((n, size), dtype=torch.uint8, device="cuda")
    where = torch.arange(1 << 20, size - 8, 1 << 20, device="cuda")
    for s in range(n):
        for j, b in enumerate(b"needle"):
            d[s, where + j + s] = b
    A, _ = automaton("bytes", False, [list(b"needle"), list(b"eed"), list(b"le\0")])
    want = rows(A.find_leftmost_longest_batch(d))
    cut = (1 << 20) * 7 + 3                                 # inside a planted key
    feeds = [(d[:, :cut].contiguous(), None), (d[:, cut:].contiguous(), None)]
    del d
    torch.cuda.empty_cache()
    got = _collect(A.stream_batch(n, leftmost_longest=True), feeds, n)
    assert len(want) > 2000 and np.array_equal(got, want)


@pytest.mark.gpu
def test_gpu_capacity_contract():
    """caps 0, 1 and n-1 for records and output bytes, on the host and the device entries: nothing is committed, and the
    repeated feed gives the answer of a batch that never overflowed"""
    import torch
    keys = [b"ab", b"b", b"abc", b"ca"]
    A, _ = automaton("bytes", False, keys)
    table = {b"ab": b"XYZW", b"b": b"", b"abc": b"q", b"ca": b"CA!"}
    R = A.replacer(table)
    chunks = [b"abcabxbab" * 5, b"bbbbca", b"zzab", b"c"]
    tb, flat, offs = table_and_batch(A, chunks)
    L = N.lib()
    r = R._replacer(tb, False, 0)
    prime = [b"a", b"", b"", b"xab"]

    def fresh(kind):
        B = A.stream_batch(4, leftmost_longest=True) if kind == "find" else R.stream_batch(4)
        B.feed(prime)
        return B

    ref = fresh("find").feed(chunks)
    n = len(ref)
    ref_out = fresh("replace").feed(chunks)
    total = sum(len(x) for x in ref_out)
    assert n > 3 and total > 3
    for cap in (0, 1, n - 1):
        B = fresh("find")
        found = ctypes.c_int64(0)
        assert L.acb_streams_feed_leftmost_host(B._ss, tb, N.ptr(flat), flat.size, N.ptr(offs), 4, 0, None, 0, None, cap,
                                                ctypes.byref(found), 0) == N.ACB_EOVERFLOW and found.value == n
        assert list(B.positions) == [1, 0, 0, 3]
        d = torch.from_numpy(flat.copy()).cuda()
        d_off = torch.from_numpy(offs).cuda()
        out = torch.zeros((max(cap, 1), 3), dtype=torch.int32, device="cuda")
        cnt = torch.zeros(1, dtype=torch.int64, device="cuda")
        assert L.acb_streams_feed_leftmost_device(B._ss, tb, d.data_ptr(), flat.size, d_off.data_ptr(), 4, 0, None, 0, out.data_ptr(),
                                                  cap, cnt.data_ptr(), torch.cuda.current_stream().cuda_stream, 0) == N.ACB_OK
        assert int(cnt.item()) == n and list(B.positions) == [1, 0, 0, 3]
        m = B.feed(chunks)
        assert np.array_equal(m.hay_id, ref.hay_id) and np.array_equal(m.end_index, ref.end_index)
        S = fresh("replace")
        oo = np.zeros(5, np.int64)
        t = ctypes.c_int64(0)
        buf = np.full(cap + 16, 0xEE, np.uint8)
        assert L.acb_streams_replace_host(S._ss, r, tb, N.ptr(flat), flat.size, N.ptr(offs), 4, 0, None, 0, 0, N.ptr(oo), N.ptr(buf),
                                          cap, ctypes.byref(t)) == N.ACB_EOVERFLOW and t.value == total
        assert (buf == 0xEE).all() and list(S.positions) == [1, 0, 0, 3]
        dout = torch.full((cap + 16,), 0xEE, dtype=torch.uint8, device="cuda")
        doo = torch.zeros(5, dtype=torch.int64, device="cuda")
        tt = torch.zeros(1, dtype=torch.int64, device="cuda")
        assert L.acb_streams_replace_device(S._ss, r, tb, d.data_ptr(), flat.size, d_off.data_ptr(), 4, 0, None, 0, doo.data_ptr(),
                                            dout.data_ptr(), cap, tt.data_ptr(), torch.cuda.current_stream().cuda_stream, 0) == N.ACB_OK
        assert int(tt.item()) == total and bool((dout == 0xEE).all()) and list(S.positions) == [1, 0, 0, 3]
        assert S.feed(chunks) == ref_out
    F = A.stream_batch(2)
    found = ctypes.c_int64(0)
    assert L.acb_streams_feed_leftmost_host(F._ss, tb, N.ptr(flat), 4, None, 1, 4, None, 0, None, 8, ctypes.byref(found), 0) == N.ACB_EINVAL
    B = A.stream_batch(2, leftmost_longest=True)
    assert L.acb_streams_feed_host(B._ss, tb, N.ptr(flat), 4, None, 1, 4, None, None, 8, ctypes.byref(found), 0, 1) == N.ACB_EINVAL


@pytest.mark.gpu
@pytest.mark.parametrize("fl", ["bytes", "unicode"])
def test_gpu_cuda_tensors_on_a_side_stream(fl):
    import torch
    rng = np.random.default_rng(21)
    case = "bytes" if fl == "bytes" else "wide"
    fl, seq, al = CASES[case]
    keys = sorted({tuple(int(x) for x in rng.choice(al[:2], size=int(rng.integers(1, 5)))) for _ in range(10)})
    A, O = automaton(fl, seq, keys)
    reps = replace_reps(case, keys, rng)
    R = A.replacer({obj(fl, seq, k): obj(fl, seq, r) for k, r in zip(keys, reps)})
    texts = [[int(x) for x in rng.choice(al, size=28)] for _ in range(300)]
    host = np.stack([np.asarray(t, dtype=DT[A._L]).view(np.uint8) for t in texts])
    d = torch.from_numpy(host).cuda()
    W = 7 * A._L
    views = {"whole": (lambda i: d[:, i * W:(i + 1) * W].contiguous(), texts)}
    if A._L == 1:
        zero = torch.zeros((1, W), dtype=torch.uint8, device="cuda")   # rows of 7 bytes: row 1 starts off a 16-byte boundary
        views["misaligned"] = (lambda i: torch.cat([zero, d[:, i * W:(i + 1) * W]])[1:], texts)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    for name, (piece, ts) in views.items():
        B = A.stream_batch(len(ts), leftmost_longest=True)
        S = R.stream_batch(len(ts))
        got = [[] for _ in ts]
        outs = []
        with torch.cuda.stream(side):
            for i in range(4):
                t = piece(i)
                if name == "misaligned":
                    assert t.data_ptr() % 16 != 0
                m = B.feed(t)
                for h, e, v in zip(m.hay_id.tolist(), m.end_index.tolist(), m.values()):
                    got[h].append((e, v))
                outs.append(S.feed(t))
            m = B.finish()
            rest = S.finish()
        side.synchronize()
        for h, e, v in zip(m.hay_id.tolist(), m.end_index.tolist(), m.values()):
            got[h].append((e, v))
        assert all(o.is_cuda and f.is_cuda for o, f in outs)
        parts = [split(o.cpu().numpy(), f.cpu().numpy(), A._L) for o, f in outs]
        for s, t in enumerate(ts):
            assert got[s] == _want_matches(O, keys, t, case), name
            out = [x for p in parts for x in p[s]]
            assert out + _letters(case, rest[s]) == _want_output(O, keys, t, reps, case), name


@pytest.mark.gpu
def test_gpu_interleaved_with_other_calls_on_one_table():
    """feeds between find_leftmost_longest_batch, replace_batch and a find_all stream batch on the same table"""
    rng = np.random.default_rng(33)
    keys = [b"ab", b"abc", b"bc", b"cab", b"a"]
    A, O = automaton("bytes", False, keys)
    texts = [bytes(rng.choice(list(b"abc"), size=90).astype(np.uint8)) for _ in range(50)]
    R = A.replacer({k: k.upper() * 2 for k in keys})
    B = A.stream_batch(50, leftmost_longest=True)
    S = R.stream_batch(50)
    F = A.stream_batch(50)
    whole = rows(A.find_leftmost_longest_batch(texts))
    wout = R.replace_batch(texts)
    recs, outs, fa = [], [b""] * 50, 0
    for i in range(0, 90, 13):
        chunks = [t[i:i + 13] for t in texts]
        recs.append(rows(B.feed(chunks)))
        assert rows(A.find_leftmost_longest_batch(texts)).tolist() == whole.tolist()
        outs = [a + b for a, b in zip(outs, S.feed(chunks))]
        assert R.replace_batch(texts) == wout
        fa += len(F.feed(chunks))
    recs.append(rows(B.finish()))
    r = np.concatenate(recs)
    assert np.array_equal(r[np.lexsort((r[:, 1], r[:, 0]))], whole)
    assert [a + b for a, b in zip(outs, S.finish())] == wout
    assert fa == len(A.find_all_batch(texts))
