"""stream_batch(whole_words=...) for find_all, leftmost-longest and replacing streams: whole-word matches chunk by chunk.

Whatever the chunking, a stream's feeds plus its finish must give exactly what the whole-batch methods give for its whole
text with the same word set: emul_words.definition over the C oracle's full list, then emul_leftmost.greedy or
emul_replace.definition (CPU and small GPU cases), or find_all_batch / find_leftmost_longest_batch / replace_batch of the
whole text on the GPU (at scale).  The CPU tests run the Python layer on the restatement of the native feeds
(tests/emul_stream_words.py); the gpu-marked tests run the real kernels."""
import ctypes
import re

import numpy as np
import pytest

import emul_leftmost
import emul_replace
import emul_stream_leftmost
import emul_stream_words
import emul_streams
import emul_words
import pyahocorasick_b200 as pkg
from batch_cases import CASES, DT, automaton, fake_table, obj, oracle_full, rows, skip_if_device, table_and_batch
from pyahocorasick_b200 import _native as N

FUZZ_CASES = ["bytes", "latin1", "wide", "mixed"]           # every case but the key sequences
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
    return [True, b"", b"a_ "] if CASES[case][0] == "bytes" else [True, "", "ał_\U0001F600"]


def _alphabet(case):
    return CASES[case][2] + [SPACE, UNDERSCORE]


def _key_sets(case, rng):
    """random keys over the alphabet with space and underscore, the new / new york pair, and T = 0"""
    al = _alphabet(case)
    yield sorted({tuple(int(x) for x in rng.choice(al, size=int(rng.integers(1, 6)))) for _ in range(int(rng.integers(1, 8)))})
    yield [list(b"ab"), list(b"ab a"), list(b"b"), list(b"a")]
    yield sorted({(int(x),) for x in rng.choice(al, size=2)})                             # T = 0


def _texts(case, keys, rng, n):
    """per stream, a list of segments (texts between finishes)"""
    al = _alphabet(case)
    out = []
    for _ in range(n):
        segs = []
        for _ in range(int(rng.integers(1, 3))):
            r = int(rng.integers(0, 4))
            if r == 0:
                segs.append([])
            elif r == 1:
                segs.append(list(keys[int(rng.integers(0, len(keys)))]))                # one key: both edges
            else:
                body = []
                while len(body) < int(rng.integers(1, 60)):
                    body += list(keys[int(rng.integers(0, len(keys)))]) if rng.integers(0, 2) else \
                        [int(x) for x in rng.choice(al, size=int(rng.integers(1, 4)))]
                segs.append(body)
        out.append(segs)
    return out


def _chunk_len(T, rng):
    return int(rng.choice([0, 1, max(T, 1), T + 1, T + 2, 3 * T + 1, int(rng.integers(1, 20))]))


def _drive(case, texts, rng, feed, finish, T, check_lag=None, reset=None):
    """Feed every stream's segments in random chunks: each call takes a random subset of the streams, in random order,
    and an exhausted segment is finished in that call or a later one (empty chunks may come in between).  reset(ids),
    when given, sometimes restarts a stream mid-segment: the segment then starts over.  feed(chunks, ids) / finish(ids)
    return per id what it released.  Returns per stream and segment the releases.  check_lag(stream, segment,
    position) runs after every feed."""
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
        if reset is not None and rng.integers(0, 12) == 0:
            s = pick[0]
            reset([s])
            got[s][seg[s]] = []
            off[s] = 0
            continue
        done = [s for s in pick if off[s] >= len(texts[s][seg[s]]) and rng.integers(0, 3)]
        if done:
            for s, r in zip(done, finish(done)):
                got[s][seg[s]].append(r)
                seg[s] += 1
                off[s] = 0


def _per_id(m, ids):
    return [[(int(e), int(v)) for h, e, v in zip(m.hay_id.tolist(), m.end_index.tolist(), m.values()) if h == s] for s in ids]


def _letters(case, item):
    if CASES[case][1]:
        return list(item)
    return list(item) if isinstance(item, bytes) else [ord(c) for c in item]


def _want(O, keys, text, case, words):
    """(find_all, leftmost-longest) of one whole text by the definitions: [(end, key)]"""
    kl = [len(k) for k in keys]
    kept = emul_words.definition([text], oracle_full(O, [text], case), kl, _is_word(case, words))
    return [(e, k) for _, e, k in kept], [(e, k) for _, e, k in emul_leftmost.greedy(kept, kl)]


def _reps(case, keys, rng):
    al = _alphabet(case)
    return [[int(x) for x in rng.choice(al, size=int(rng.integers(0, 4)))] for _ in keys]


def _run_case(case, keys, texts, rng, algo, words, emulated):
    fl, seq, _ = CASES[case]
    A, O = automaton(fl, seq, keys)
    T = max(len(k) for k in keys) - 1
    kl = [len(k) for k in keys]
    for leftmost in (False, True):
        B = A.stream_batch(len(texts), leftmost_longest=leftmost, algo=algo, whole_words=words)
        got_now = [[] for _ in texts]

        def lag(s, g, p):
            want_all, want_ll = _want(O, keys, texts[s][g][:p] + [SPACE], case, words)     # what the text decides by p
            seen = {x for r in got_now[s] for x in r}
            if leftmost:
                full = _want(O, keys, texts[s][g], case, words)[1]
                assert {x for x in full if x[0] - kl[x[1]] + 1 < p - T - 1} <= seen, (case, keys, texts[s][g], p)
            else:
                assert {x for x in want_all if x[0] <= p - 2} <= seen, (case, keys, texts[s][g], p)
            if emulated:
                assert len(B._ss["held"][s]) // A._L <= T + 1

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

        def reset(ids):
            B.reset(ids)
            for s in ids:
                got_now[s].clear()

        got = _drive(case, texts, rng, feed, finish, T, lag, reset)
        for s, segs in enumerate(texts):
            for g, text in enumerate(segs):
                want = _want(O, keys, text, case, words)[int(leftmost)]
                assert [x for r in got[s][g] for x in r] == want, (case, algo, leftmost, keys, text, words)
        assert not B.positions.any()
    reps = _reps(case, keys, rng)
    R = A.replacer({obj(fl, seq, k): obj(fl, seq, r) for k, r in zip(keys, reps)})
    S = R.stream_batch(len(texts), algo=algo, whole_words=words)
    got = _drive(case, texts, rng, lambda c, i: [_letters(case, x) for x in S.feed(c, i)],
                 lambda i: [_letters(case, x) for x in S.finish(i)], T)
    for s, segs in enumerate(texts):
        for g, text in enumerate(segs):
            want = emul_replace.definition(text, _want(O, keys, text, case, words)[1], kl, reps)
            assert [x for r in got[s][g] for x in r] == want, (case, algo, keys, text, reps, words)


def _fuzz(algo, emulated, seed, rounds):
    rng = np.random.default_rng(seed)
    for case in FUZZ_CASES:
        for words in _word_sets(case):
            for _ in range(rounds):
                for keys in _key_sets(case, rng):
                    _run_case(case, [list(k) for k in keys], _texts(case, keys, rng, int(rng.integers(1, 5))), rng, algo,
                              words, emulated)


# ------------------------------------------------------------------ the Python layer on the restatement (CPU)
def test_python_layer_on_the_restatement(monkeypatch):
    """both flavours, latin-1 / wide / mixed chunks; True, custom and empty word sets; chunks of 0, 1, T, T+1, T+2 and
    3T+1 letters, None chunks, streams left out of a call, reset and finish mid-stream"""
    emul_stream_words.install(monkeypatch)
    _fuzz("auto", True, 5, 2)


NEW = ["new", "new york"]


@pytest.mark.parametrize("leftmost", [False, True])
def test_new_york_split_at_every_position(monkeypatch, leftmost):
    """`new` is found in `new yorker`, `new york` is not: the letter after it is a word letter, also when it arrives in
    a later chunk; both split at every position, and fed letter by letter"""
    emul_stream_words.install(monkeypatch)
    mod = pkg.flavour("bytes")
    A = mod.Automaton(mod.STORE_INTS)
    for i, k in enumerate(NEW):
        A.add_word(k.encode(), i)
    A.make_automaton()
    text = b"new yorker"
    B = A.stream_batch(1, leftmost_longest=leftmost, whole_words=True)
    for cut in range(len(text) + 1):
        got = []
        for piece in (text[:cut], text[cut:]):
            m = B.feed([piece])
            got += list(zip(m.end_index.tolist(), m.values()))
        m = B.finish()
        assert got + list(zip(m.end_index.tolist(), m.values())) == [(2, 0)], cut
    ends = [B.feed([bytes([piece])]).end_index.tolist() for piece in text] + [B.finish().end_index.tolist()]
    assert sum(ends, []) == [2] and ends[8 if leftmost else 3] == [2]       # start 0 < 9 - T - 1; end 2 <= 4 - 2
    R = A.replacer({b"new": b"NEW", b"new york": b"NYC"})
    S = R.stream_batch(1, whole_words=True)
    for cut in range(len(text) + 1):
        out = S.feed([text[:cut]])[0] + S.feed([text[cut:]])[0] + S.finish()[0]
        assert out == b"NEW yorker", cut
    assert S.feed([b"new york!"]) == [b"NYC"] and S.finish() == [b"!"]     # `!` decides `new york`; it is held back
    assert S.feed([b"new york"]) == [b""] and S.finish() == [b"NYC"]


def test_left_neighbour_from_an_earlier_feed(monkeypatch):
    """`abc` after `z` (not a whole word) and after a space (a whole word), where that letter arrived three feeds before
    the match is decided: only the stream's left-neighbour byte knows it"""
    emul_stream_words.install(monkeypatch)
    A, _ = automaton("bytes", False, [list(b"abc")])
    feeds = [(b"z", b" "), (b"ab", b"ab"), (b"c", b"c"), (b" ", b" ")]
    for leftmost in (False, True):
        B = A.stream_batch(2, leftmost_longest=leftmost, whole_words=True)
        got = [B.feed([a, b]).hay_id.tolist() for a, b in feeds]
        assert B.positions.tolist() == [5, 5]
        if not leftmost:
            assert got == [[], [], [], [1]]              # reported by the feed that brought the space after it
        assert sum(got, []) + B.finish().hay_id.tolist() == [1], (leftmost, got)
    S = A.replacer({b"abc": b"X"}).stream_batch(2, whole_words=True)
    outs = [S.feed([a, b]) for a, b in feeds]
    fin = S.finish()
    assert [b"".join(o[i] for o in outs) + fin[i] for i in range(2)] == [b"zabc ", b" X "]


def test_refusals_and_finish_of_plain_batches(monkeypatch):
    emul_streams.install(monkeypatch)
    emul_stream_leftmost.install(monkeypatch)
    emul_stream_words.install(monkeypatch)
    mod = pkg.flavour("bytes")
    A = mod.Automaton()
    A.add_word(b"ab", b"X")
    A.make_automaton()
    for kw in ({"long": True}, {"ignore_white_space": True}, {"long": True, "leftmost_longest": True}):
        with pytest.raises(ValueError):
            A.stream_batch(2, whole_words=True, **kw)
    with pytest.raises(ValueError):
        A.stream_batch(2, whole_words="ab")                   # a str set for the bytes flavour
    with pytest.raises(TypeError):
        A.stream_batch(2, whole_words=3)
    with pytest.raises(ValueError):
        A.replacer().stream_batch(2, whole_words="ab")
    with pytest.raises(ValueError):
        A.stream_batch(2).finish()                           # finish still belongs to word and leftmost batches
    S = mod.Automaton(mod.STORE_ANY, mod.KEY_SEQUENCE)
    S.add_word((1, 2), 0)
    S.make_automaton()
    with pytest.raises(ValueError):
        S.stream_batch(1, whole_words=True)
    B = A.stream_batch(2, whole_words=True)
    assert B.whole_words and not B.leftmost_longest
    assert len(B.feed([b"xab", b"ab"])) == 0                 # "xab" is one word; "ab" of stream 1 waits for its right neighbour
    assert B.finish([1]).hay_id.tolist() == [1] and B.positions.tolist() == [3, 0]
    P = A.stream_batch(2, whole_words=False)                 # False: the plain find_all batch of today
    assert not P.whole_words and len(P.feed([b"xab", b"ab"])) == 2
    A.add_word(b"cd", b"Y")
    for call in (lambda: B.feed([b"a"]), lambda: B.finish(), lambda: B.reset()):
        with pytest.raises(ValueError):
            call()


def test_c_entries_check_arguments_first():
    L = N.lib()
    ss = ctypes.c_void_p()
    cnt = np.zeros(4, np.int64)
    hay = np.zeros(32, np.uint8)
    bits = np.zeros(8, np.uint32)
    assert L.acb_streams_new_words(None, 1, 0, None, 0, ctypes.byref(ss)) == N.ACB_EINVAL
    fake = fake_table(1)
    assert L.acb_streams_new_words(ctypes.addressof(fake), 1, 0, N.ptr(bits), 257, ctypes.byref(ss)) == N.ACB_EINVAL
    assert L.acb_streams_new_words(ctypes.addressof(fake), 1, 1, None, 8, ctypes.byref(ss)) == N.ACB_EINVAL
    assert L.acb_streams_new_words(ctypes.addressof(fake), 1, 0, N.ptr(bits), -1, ctypes.byref(ss)) == N.ACB_EINVAL
    assert L.acb_streams_feed_words_device(None, None, None, 0, None, 0, 0, None, 0, None, 0, N.ptr(cnt), None, 0) == N.ACB_EINVAL
    found = ctypes.c_int64(0)
    assert L.acb_streams_feed_words_host(None, None, N.ptr(hay), 32, None, 1, 32, None, 0, None, 0, ctypes.byref(found), 0) == N.ACB_EINVAL


def test_c_entries_fail_loudly_without_a_device():
    skip_if_device()
    ss = ctypes.c_void_p()
    for L_ in (1, 2, 4):
        fake = fake_table(L_)
        assert N.lib().acb_streams_new_words(ctypes.addressof(fake), 4, 1, None, 0, ctypes.byref(ss)) == N.ACB_ECUDA
        assert N.last_error()


# ------------------------------------------------------------------ the real kernels
@pytest.mark.gpu
@pytest.mark.parametrize("algo", ["filter", "dfa"])
def test_gpu_fuzz_against_the_definition(algo):
    _fuzz(algo, False, 11 if algo == "filter" else 12, 1)


def _collect(B, feeds):
    """run B.feed over [(tensor or array, ids)] and finish -> int64 records (stream, end, key id), stable-sorted by stream"""
    recs = []
    for batch, ids in feeds:
        recs.append(rows(B.feed(batch, ids)))
    recs.append(rows(B.finish()))
    r = np.concatenate(recs)
    return r[np.argsort(r[:, 0], kind="stable")]


def _by_stream(r):
    return r[np.argsort(r[:, 0], kind="stable")]


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


C2_WORDS = b"abcdefghijklmnopqrstuvwxyz"


@pytest.mark.gpu
@pytest.mark.parametrize("step", [256, 1, 7, 64])
def test_gpu_c2_million_streams(step):
    """10^6 streams of the C2 key set (one planted key per 256-byte row) fed `step` letters at a time, under the word set
    of the lowercase letters: a planted key survives when neither neighbour is lowercase, which holds for 33.9 % of them
    (counted below on the CPU).  Against find_all_batch, find_leftmost_longest_batch and replace_batch of the whole rows."""
    import torch
    from pyahocorasick_b200 import synth
    w = synth.make("C2")
    A = synth.build_automaton(w.keys)
    n = w.n_hay
    hay = w.haystacks
    low = np.zeros(256, dtype=bool)
    low[np.frombuffer(C2_WORDS, dtype=np.uint8)] = True
    kl = np.array([len(k) for k in w.keys])
    end, start = w.planted_end, w.planted_end - kl[w.planted_key] + 1
    lw = (start > 0) & low[hay[w.planted_hay, np.maximum(start - 1, 0)]]
    rw = (end < hay.shape[1] - 1) & low[hay[w.planted_hay, np.minimum(end + 1, hay.shape[1] - 1)]]
    share = float((~lw & ~rw).mean())
    assert 0.3 < share < 0.38
    d = torch.from_numpy(hay).cuda()
    feeds = [(d[:, i:i + step].contiguous(), None) for i in range(0, d.shape[1], step)]
    want_all = rows(A.find_all_batch(d, whole_words=C2_WORDS))
    want_ll = rows(A.find_leftmost_longest_batch(d, whole_words=C2_WORDS))
    planted = set(zip(w.planted_hay[~lw & ~rw].tolist(), w.planted_end[~lw & ~rw].tolist()))
    assert planted <= set(zip(want_all[:, 0].tolist(), want_all[:, 1].tolist()))
    assert np.array_equal(_collect(A.stream_batch(n, whole_words=C2_WORDS), feeds), want_all)
    assert np.array_equal(_collect(A.stream_batch(n, leftmost_longest=True, whole_words=C2_WORDS), feeds), want_ll)
    rng = np.random.default_rng(step)
    table = {k: bytes(rng.integers(0x41, 0x5B, size=int(rng.integers(0, 20)), dtype=np.uint8)) for k in w.keys}
    R = A.replacer(table)
    wout, woffs = R.replace_batch(d, whole_words=C2_WORDS)
    S = R.stream_batch(n, whole_words=C2_WORDS)
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
    keys = sorted({bytes(rng.choice(list(b"ab "), size=int(rng.integers(1, klen + 1))).astype(np.uint8)) for _ in range(8)}
                  | {bytes(rng.choice(list(b"ab "), size=klen).astype(np.uint8))})
    A, _ = automaton("bytes", False, keys)
    n = 6
    texts = []
    for _ in range(n):
        t = b""
        while len(t) < 3 * klen:
            t += keys[int(rng.integers(0, len(keys)))] if rng.integers(0, 2) else bytes(rng.choice(list(b"ab c"), size=5).astype(np.uint8))
        texts.append(t)
    want_all = _by_stream(rows(A.find_all_batch(texts, whole_words=b"ab")))
    want_ll = rows(A.find_leftmost_longest_batch(texts, whole_words=b"ab"))
    assert len(want_ll) > 0
    R = A.replacer({k: k[: len(k) // 3] for k in keys})
    wout = R.replace_batch(texts, whole_words=b"ab")
    F = A.stream_batch(n, whole_words=b"ab")
    B = A.stream_batch(n, leftmost_longest=True, whole_words=b"ab")
    S = R.stream_batch(n, whole_words=b"ab")
    pos = [0] * n
    feeds, outs = [], [b""] * n
    while any(p < len(t) for p, t in zip(pos, texts)):
        chunks = []
        for s in range(n):
            k = int(rng.choice([1, klen - 1, klen, klen + 1, klen + 2, 3 * klen]))
            chunks.append(texts[s][pos[s]:pos[s] + k])
            pos[s] += k
        feeds.append((chunks, None))
        outs = [a + b for a, b in zip(outs, S.feed(chunks))]
    assert np.array_equal(_collect(F, feeds), want_all)
    assert np.array_equal(_collect(B, feeds), want_ll)
    assert [a + b for a, b in zip(outs, S.finish())] == wout


@pytest.mark.gpu
def test_gpu_staged_batch_past_2_gib():
    """two chunks of 1.1 GB each: the staged batch passes 2^31 bytes; planted keys cross the feeds' boundary, half of them
    inside a word"""
    import torch
    n, size = 2, 1_100_000_000
    d = torch.full((n, size), 0x20, dtype=torch.uint8, device="cuda")
    where = torch.arange(1 << 20, size - 8, 1 << 20, device="cuda")
    for s in range(n):
        for j, b in enumerate(b"needle"):
            d[s, where + j + s] = b
        d[s, where[::2] + s + 6] = ord("s")                  # "needles": not a whole word
    A, _ = automaton("bytes", False, [list(b"needle"), list(b"eed"), list(b"le ")])
    want_all = _by_stream(rows(A.find_all_batch(d, whole_words=True)))
    want_ll = rows(A.find_leftmost_longest_batch(d, whole_words=True))
    cut = (1 << 20) * 7 + 3                                 # inside a planted key
    feeds = [(d[:, :cut].contiguous(), None), (d[:, cut:].contiguous(), None)]
    del d
    torch.cuda.empty_cache()
    assert len(want_ll) > 1000 and np.array_equal(_collect(A.stream_batch(n, leftmost_longest=True, whole_words=True), feeds), want_ll)
    assert np.array_equal(_collect(A.stream_batch(n, whole_words=True), feeds), want_all)


@pytest.mark.gpu
def test_gpu_capacity_contract():
    """capacities 0, 1, n-1 and n for records and output bytes on all six entries a word batch takes: below n nothing is
    committed, and the repeated feed gives the answer of a batch that never overflowed"""
    import torch
    keys = [b"ab", b"b", b"abc", b"ca"]
    A, _ = automaton("bytes", False, keys)
    R = A.replacer({b"ab": b"XYZW", b"b": b"", b"abc": b"q", b"ca": b"CA!"})
    chunks = [b"ab ab b abc " * 5, b"b b ca ", b"zz ab", b" c"]
    tb, flat, offs = table_and_batch(A, chunks)
    L = N.lib()
    r = R._replacer(tb, False, 0)
    prime = [b"a", b"", b"", b"x ab"]
    stream = torch.cuda.current_stream().cuda_stream
    d = torch.from_numpy(flat.copy()).cuda()
    d_off = torch.from_numpy(offs).cuda()

    def fresh(kind):
        B = R.stream_batch(4, whole_words=True) if kind == "replace" else \
            A.stream_batch(4, leftmost_longest=kind == "leftmost", whole_words=True)
        B.feed(prime)
        return B

    for kind, host, dev in (("find_all", L.acb_streams_feed_words_host, L.acb_streams_feed_words_device),
                            ("leftmost", L.acb_streams_feed_leftmost_host, L.acb_streams_feed_leftmost_device)):
        ref = fresh(kind).feed(chunks)
        n = len(ref)
        assert n > 3
        want = np.stack([ref.hay_id, ref.end_index - np.array([1, 0, 0, 4])[ref.hay_id], ref.key_id.astype(np.int64)], axis=1)
        for cap in (0, 1, n - 1, n):
            B = fresh(kind)
            found = ctypes.c_int64(0)
            out = np.zeros(max(cap, 1), dtype=N.MATCH_DTYPE)
            rc = host(B._ss, tb, N.ptr(flat), flat.size, N.ptr(offs), 4, 0, None, 0, N.ptr(out), cap, ctypes.byref(found), 0)
            assert found.value == n and rc == (N.ACB_OK if cap == n else N.ACB_EOVERFLOW), (kind, cap)
            D = fresh(kind)
            dout = torch.full((max(cap, 1), 3), -7, dtype=torch.int32, device="cuda")
            cnt = torch.zeros(1, dtype=torch.int64, device="cuda")
            assert dev(D._ss, tb, d.data_ptr(), flat.size, d_off.data_ptr(), 4, 0, None, 0, dout.data_ptr(), cap,
                       cnt.data_ptr(), stream, 0) == N.ACB_OK
            assert int(cnt.item()) == n
            if cap == n:
                got = np.stack([out["hay_id"], out["end_index"], out["key_id"]], axis=1).astype(np.int64)
                assert np.array_equal(got, want) and np.array_equal(dout.cpu().numpy().astype(np.int64), want), kind
                assert list(B.positions) == list(D.positions) == [1 + len(chunks[0]), len(chunks[1]), len(chunks[2]), 4 + len(chunks[3])]
                continue
            for X in (B, D):                                 # nothing committed: the same feed again gives the reference
                assert list(X.positions) == [1, 0, 0, 4]
                m = X.feed(chunks)
                assert np.array_equal(m.hay_id, ref.hay_id) and np.array_equal(m.end_index, ref.end_index), (kind, cap)
    ref_out = fresh("replace").feed(chunks)
    total = sum(len(x) for x in ref_out)
    for cap in (0, 1, total - 1):
        S = fresh("replace")
        oo = np.zeros(5, np.int64)
        t = ctypes.c_int64(0)
        buf = np.full(cap + 16, 0xEE, np.uint8)
        assert L.acb_streams_replace_host(S._ss, r, tb, N.ptr(flat), flat.size, N.ptr(offs), 4, 0, None, 0, 0, N.ptr(oo), N.ptr(buf),
                                          cap, ctypes.byref(t)) == N.ACB_EOVERFLOW and t.value == total
        assert (buf == 0xEE).all() and list(S.positions) == [1, 0, 0, 4]
        dout = torch.full((cap + 16,), 0xEE, dtype=torch.uint8, device="cuda")
        doo = torch.zeros(5, dtype=torch.int64, device="cuda")
        tt = torch.zeros(1, dtype=torch.int64, device="cuda")
        assert L.acb_streams_replace_device(S._ss, r, tb, d.data_ptr(), flat.size, d_off.data_ptr(), 4, 0, None, 0, doo.data_ptr(),
                                            dout.data_ptr(), cap, tt.data_ptr(), stream, 0) == N.ACB_OK
        assert int(tt.item()) == total and bool((dout == 0xEE).all()) and list(S.positions) == [1, 0, 0, 4]
        assert S.feed(chunks) == ref_out
    S = fresh("replace")
    oo = np.zeros(5, np.int64)
    t = ctypes.c_int64(0)
    buf = np.zeros(total + 16, np.uint8)
    assert L.acb_streams_replace_host(S._ss, r, tb, N.ptr(flat), flat.size, N.ptr(offs), 4, 0, None, 0, 0, N.ptr(oo), N.ptr(buf),
                                      total, ctypes.byref(t)) == N.ACB_OK and t.value == total
    assert b"".join(ref_out) == buf[:total].tobytes()
    S = fresh("replace")
    dout = torch.zeros(total + 16, dtype=torch.uint8, device="cuda")
    doo = torch.zeros(5, dtype=torch.int64, device="cuda")
    tt = torch.zeros(1, dtype=torch.int64, device="cuda")
    assert L.acb_streams_replace_device(S._ss, r, tb, d.data_ptr(), flat.size, d_off.data_ptr(), 4, 0, None, 0, doo.data_ptr(),
                                        dout.data_ptr(), total, tt.data_ptr(), stream, 0) == N.ACB_OK
    assert int(tt.item()) == total and dout[:total].cpu().numpy().tobytes() == b"".join(ref_out)
    # each feed refuses the batches of the other kinds
    F = A.stream_batch(4, whole_words=True)
    W = A.stream_batch(4, leftmost_longest=True, whole_words=True)
    P = A.stream_batch(4, leftmost_longest=True)
    found = ctypes.c_int64(0)
    args = (tb, N.ptr(flat), 4, None, 1, 4, None, 0, None, 8, ctypes.byref(found), 0)
    assert L.acb_streams_feed_words_host(W._ss, *args) == N.ACB_EINVAL
    assert L.acb_streams_feed_words_host(P._ss, *args) == N.ACB_EINVAL
    assert L.acb_streams_feed_leftmost_host(F._ss, *args) == N.ACB_EINVAL
    assert L.acb_streams_feed_host(F._ss, tb, N.ptr(flat), 4, None, 1, 4, None, None, 8, ctypes.byref(found), 0, 1) == N.ACB_EINVAL
    assert L.acb_streams_feed_host(W._ss, tb, N.ptr(flat), 4, None, 1, 4, None, None, 8, ctypes.byref(found), 0, 1) == N.ACB_EINVAL
    bad = np.array([0, 3, 2, 4, flat.size], np.int64)
    assert L.acb_streams_feed_words_host(F._ss, tb, N.ptr(flat), flat.size, N.ptr(bad), 4, 0, None, 0, None, 8, ctypes.byref(found), 0) == N.ACB_EINVAL
    ids = np.array([0, 0], np.int32)
    assert L.acb_streams_feed_words_host(F._ss, tb, N.ptr(flat), 4, None, 2, 2, N.ptr(ids), 0, None, 8, ctypes.byref(found), 0) == N.ACB_EINVAL
    assert not F.positions.any()


@pytest.mark.gpu
@pytest.mark.parametrize("fl", ["bytes", "unicode"])
def test_gpu_cuda_tensors_on_a_side_stream(fl):
    import torch
    rng = np.random.default_rng(21)
    case = "bytes" if fl == "bytes" else "wide"
    fl, seq, _ = CASES[case]
    al = _alphabet(case)
    keys = sorted({tuple(int(x) for x in rng.choice(al[:2] + [SPACE], size=int(rng.integers(1, 5)))) for _ in range(10)})
    A, O = automaton(fl, seq, keys)
    kl = [len(k) for k in keys]
    reps = _reps(case, keys, rng)
    R = A.replacer({obj(fl, seq, k): obj(fl, seq, r) for k, r in zip(keys, reps)})
    texts = [[int(x) for x in rng.choice(al, size=28)] for _ in range(300)]
    host = np.stack([np.asarray(t, dtype=DT[A._L]).view(np.uint8) for t in texts])
    d = torch.from_numpy(host).cuda()
    W = 7 * A._L
    views = {"whole": lambda i: d[:, i * W:(i + 1) * W].contiguous()}
    if A._L == 1:
        zero = torch.zeros((1, W), dtype=torch.uint8, device="cuda")   # rows of 7 bytes: row 1 starts off a 16-byte boundary
        views["misaligned"] = lambda i: torch.cat([zero, d[:, i * W:(i + 1) * W]])[1:]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    for name, piece in views.items():
        F = A.stream_batch(len(texts), whole_words=True)
        B = A.stream_batch(len(texts), leftmost_longest=True, whole_words=True)
        S = R.stream_batch(len(texts), whole_words=True)
        got = {"all": [[] for _ in texts], "ll": [[] for _ in texts]}
        outs = []
        with torch.cuda.stream(side):
            for i in range(4):
                t = piece(i)
                if name == "misaligned":
                    assert t.data_ptr() % 16 != 0
                for key, X in (("all", F), ("ll", B)):
                    m = X.feed(t)
                    for h, e, v in zip(m.hay_id.tolist(), m.end_index.tolist(), m.values()):
                        got[key][h].append((e, v))
                outs.append(S.feed(t))
            fin = {"all": F.finish(), "ll": B.finish()}
            rest = S.finish()
        side.synchronize()
        for key, m in fin.items():
            for h, e, v in zip(m.hay_id.tolist(), m.end_index.tolist(), m.values()):
                got[key][h].append((e, v))
        assert all(o.is_cuda and f.is_cuda for o, f in outs)
        parts = [[np.asarray(o.cpu().numpy()[f[i]:f[i + 1]]).view(DT[A._L]).tolist() for i in range(len(texts))]
                 for o, f in ((o, f.cpu().numpy()) for o, f in outs)]
        for s, t in enumerate(texts):
            want_all, want_ll = _want(O, keys, t, case, True)
            assert got["all"][s] == want_all and got["ll"][s] == want_ll, name
            out = [x for p in parts for x in p[s]]
            assert out + _letters(case, rest[s]) == emul_replace.definition(t, want_ll, kl, reps), name


@pytest.mark.gpu
def test_gpu_unicode_bitmap_near_the_last_code_point():
    """word letters up to U+10FFFF: the batch's 4-byte bitmap covers every code point, and a letter past the set's last
    one is never a word letter"""
    mod = pkg.flavour("unicode")
    A = mod.Automaton(mod.STORE_INTS)
    for i, k in enumerate(["ab", "\U0010FFFFa", "b\U0010FFFE"]):
        A.add_word(k, i)
    A.make_automaton()
    text = "ab\U0010FFFF ab \U0010FFFFab\U0010FFFE \U0010FFFFa b\U0010FFFE\U0010FFFF"
    for words in ("ab\U0010FFFF", "ab\U0010FFFE", True, ""):
        want_all = rows(A.find_all_batch([text], whole_words=words))
        want_ll = rows(A.find_leftmost_longest_batch([text], whole_words=words))
        for leftmost, want in ((False, want_all), (True, want_ll)):
            B = A.stream_batch(1, leftmost_longest=leftmost, whole_words=words)
            recs = [rows(B.feed([text[i:i + 3]])) for i in range(0, len(text), 3)] + [rows(B.finish())]
            assert np.array_equal(np.concatenate(recs), want), (words, leftmost)


@pytest.mark.gpu
def test_gpu_interleaved_with_other_calls_on_one_table():
    """word feeds between whole-batch word filters, plain leftmost and find_all stream batches on the same table"""
    rng = np.random.default_rng(33)
    keys = [b"ab", b"abc", b"bc", b"c a", b"a"]
    A, _ = automaton("bytes", False, keys)
    texts = [bytes(rng.choice(list(b"abc "), size=90).astype(np.uint8)) for _ in range(50)]
    R = A.replacer({k: k.upper() * 2 for k in keys})
    F = A.stream_batch(50, whole_words=True)
    B = A.stream_batch(50, leftmost_longest=True, whole_words=True)
    S = R.stream_batch(50, whole_words=True)
    P = A.stream_batch(50, leftmost_longest=True)
    Q = A.stream_batch(50)
    whole_all = _by_stream(rows(A.find_all_batch(texts, whole_words=True)))
    whole_ll = rows(A.find_leftmost_longest_batch(texts, whole_words=True))
    plain_ll = rows(A.find_leftmost_longest_batch(texts))
    wout = R.replace_batch(texts, whole_words=True)
    ra, rl, rp, outs, fa = [], [], [], [b""] * 50, 0
    for i in range(0, 90, 13):
        chunks = [t[i:i + 13] for t in texts]
        ra.append(rows(F.feed(chunks)))
        assert np.array_equal(_by_stream(rows(A.find_all_batch(texts, whole_words=True))), whole_all)
        rl.append(rows(B.feed(chunks)))
        rp.append(rows(P.feed(chunks)))
        outs = [a + b for a, b in zip(outs, S.feed(chunks))]
        assert R.replace_batch(texts, whole_words=True) == wout
        fa += len(Q.feed(chunks))
    ra.append(rows(F.finish()))
    rl.append(rows(B.finish()))
    rp.append(rows(P.finish()))
    assert np.array_equal(_by_stream(np.concatenate(ra)), whole_all)
    assert np.array_equal(_by_stream(np.concatenate(rl)), whole_ll)
    assert np.array_equal(_by_stream(np.concatenate(rp)), plain_ll)
    assert [a + b for a, b in zip(outs, S.finish())] == wout
    assert fa == len(A.find_all_batch(texts))


@pytest.mark.gpu
def test_gpu_launch_counts():
    """the launches of one feed of each kind.  The non-word feeds issue what they issued before whole-word stream
    batches existed; a leftmost word feed adds only the left-neighbour pass, and a find_all word feed stages, scans,
    flags, orders and commits"""
    keys = [b"ab", b"abc", b"bc"]
    A, _ = automaton("bytes", False, keys)
    R = A.replacer({k: b"X" for k in keys})
    chunks = [b"ab abc bc " * 3, b"abc ab"]
    L = N.lib()

    def count(B, feed=None):
        B.feed([b"a", b"b"])
        before = L.acb_launch_count()
        (feed or B.feed)(chunks)
        return L.acb_launch_count() - before

    plain = {"find_all": count(A.stream_batch(2)), "leftmost": count(A.stream_batch(2, leftmost_longest=True)),
             "replace": count(R.stream_batch(2))}
    assert plain == {"find_all": 4, "leftmost": 14, "replace": 21}
    words = {"find_all": count(A.stream_batch(2, whole_words=True)),
             "leftmost": count(A.stream_batch(2, leftmost_longest=True, whole_words=True)),
             "replace": count(R.stream_batch(2, whole_words=True))}
    # find_all: lengths, gather tiles, gather, scan, flags, sort key, emit, new X, left byte, commit
    assert words == {"find_all": 10, "leftmost": plain["leftmost"] + 1, "replace": plain["replace"] + 1}
