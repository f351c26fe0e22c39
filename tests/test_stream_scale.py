"""Stream batches at the sizes they were built for, with long keys, iter_long batches and shared table scratch.

Two references, neither of which uses the seam, gather or commit kernels:
  * the plain scan of whole streams: every stream's letters so far are kept (on the device at scale) and scanned with
    the plain find_all_batch after each feed -- a [n, len] tensor when every stream is fed and all are equally long,
    (flat, offsets) otherwise.  Its records that end at or past the stream's position before the feed are what the feed
    must return, in the same order (find_all_batch is pinned to the oracle and the reference elsewhere);
  * the C oracle per stream (long=True: the drop-in's own iter_long(c0) ... .set(ck) chain), on sampled streams.
Every mode is also fed through a twin batch in two calls whose ids are disjoint and interleaved: its records and
positions must equal the one-call batch's, which catches a lane reading or committing another stream's state."""
import ctypes

import numpy as np
import pytest

import emul
import emul_streams
import pyahocorasick_b200 as pkg
from pyahocorasick_b200 import _native as N
from pyahocorasick_b200 import synth
from batch_cases import automaton, layout
from kernel_cells import _big_batch

MiB = 1 << 20


def _arr(m):
    """a Matches as int64 rows (hay_id, end_index, key_id)"""
    return np.stack([np.asarray(m.hay_id, dtype=np.int64), np.asarray(m.end_index, dtype=np.int64),
                     np.asarray(m.key_id, dtype=np.int64)], axis=1)


def _new_part(r, before, sid):
    """plain-scan records of whole histories -> those that end at or past `before` (letters, per scanned row), with the
    row mapped to its stream id"""
    r = r[r[:, 1] >= before[r[:, 0]]]
    r[:, 0] = sid[r[:, 0]]
    return r


def _canon(r):
    """rows in (stream, end, key) order: for feeds with sort=False"""
    return r[np.lexsort((r[:, 2], r[:, 1], r[:, 0]))]


def _split_feed(Tw, chunks, ids, n_streams, **kw):
    """feed `chunks` to the twin in two calls, ids[0::2] then ids[1::2], and put the records in one-call order"""
    if ids is None:
        ids = np.arange(len(chunks), dtype=np.int64)

    def half(x):
        if isinstance(x, list):
            return x
        return np.ascontiguousarray(x) if isinstance(x, np.ndarray) else x.contiguous()
    a = Tw.feed(half(chunks[0::2]), ids[0::2], **kw)
    b = Tw.feed(half(chunks[1::2]), ids[1::2], **kw)
    r = np.concatenate([_arr(a), _arr(b)])
    rank = np.zeros(n_streams, dtype=np.int64)
    rank[ids] = np.arange(len(ids))
    return r[np.argsort(rank[r[:, 0]], kind="stable")]


# ------------------------------------------------------------------ device text
def _torch():
    import torch
    return torch


def _alnum(g, n, w):
    """uint8 [n, w] on the device, uniform over synth.ALNUM, drawn in row blocks from generator g"""
    torch = _torch()
    out = torch.empty((n, w), dtype=torch.uint8, device="cuda")
    for lo in range(0, n, 1 << 20):
        x = torch.randint(0, 62, (min(n - lo, 1 << 20), w), dtype=torch.uint8, device="cuda", generator=g)
        x += 48                                                     # 0-9
        x += (x >= 58).to(torch.uint8) * 7                          # A-Z
        x += (x >= 91).to(torch.uint8) * 6                          # a-z
        out[lo:lo + len(x)] = x
    return out


def _keymat(keys):
    torch = _torch()
    km = np.zeros((len(keys), max(map(len, keys))), dtype=np.uint8)
    for i, k in enumerate(keys):
        km[i, :len(k)] = np.frombuffer(k, dtype=np.uint8)
    return torch.from_numpy(km).cuda(), torch.tensor([len(k) for k in keys], dtype=torch.int64, device="cuda")


def _plant(text, col, keymat, klen, g, rows=None):
    """one random key per row (default: every row) across column `col`: 1 .. len-1 of its letters before it"""
    torch = _torch()
    rows = torch.arange(text.shape[0], device="cuda") if rows is None else rows
    k = torch.randint(0, len(klen), (len(rows),), device="cuda", generator=g)
    ln = klen[k]
    start = col - 1 - (torch.rand(len(rows), device="cuda", generator=g) * (ln - 1).double()).long()
    for i in range(keymat.shape[1]):
        sel = i < ln
        text[rows[sel], start[sel] + i] = keymat[k[sel], i]


def _c2():
    keys = synth.draw_keys(np.random.Generator(np.random.PCG64(1001)), synth.ALNUM, 10_000, 4, 16)   # synth.make("C2")
    return keys, synth.build_automaton(keys)


# ------------------------------------------------------------------ 1. design scale
@pytest.mark.gpu
def test_million_streams_equal_plain_scans_of_whole_streams():
    """2^20 streams, the C2 key set (T = 15), chunks of 256, 1, 7, 64 and 256 letters with a key across every boundary,
    then a host feed to a random half of the streams.  A filter batch fed in one call (once with sort=False), its twin
    fed in two calls, and a DFA batch."""
    torch = _torch()
    keys, A = _c2()
    assert A.get_stats()["longest_word"] == 16
    n, widths = 1 << 20, [256, 1, 7, 64, 256, 64]
    g = torch.Generator(device="cuda").manual_seed(2020)
    text = _alnum(g, n, sum(widths))
    km, kl = _keymat(keys)
    for col in np.cumsum(widths)[:-1].tolist():
        _plant(text, col, km, kl, g)
    S, Tw, D = A.stream_batch(n), A.stream_batch(n), A.stream_batch(n, algo="dfa")
    rng = np.random.default_rng(2020)
    P, seams = 0, 0
    for f, w in enumerate(widths):
        if f < 5:                                                   # every stream, a device tensor
            ids, sid = None, np.arange(n)
            chunks = text[:, P:P + w].contiguous()
            want = _new_part(_arr(A.find_all_batch(text[:, :P + w].contiguous())), np.full(n, P), sid)
            pos = np.full(n, P + w)
        else:                                                       # a random half, a host array
            ids = np.sort(rng.permutation(n)[:n // 2])
            sid = ids
            chunks = text[torch.from_numpy(ids).cuda(), P:P + w].cpu().numpy()
            hist = text[torch.from_numpy(ids).cuda(), :P + w].cpu().numpy()
            off = np.arange(len(ids) + 1, dtype=np.int64) * (P + w)
            want = _new_part(_arr(A.find_all_batch((hist.reshape(-1), off))), np.full(len(ids), P), sid)
            del hist
            pos = np.full(n, P)
            pos[ids] += w
        unsorted = f == 2
        got = _arr(S.feed(chunks, ids, sort=not unsorted))
        if unsorted:
            assert np.array_equal(_canon(got), _canon(want))
        else:
            assert np.array_equal(got, want)
        assert np.array_equal(_arr(D.feed(chunks, ids)), want)
        assert np.array_equal(_split_feed(Tw, chunks, ids, n), want)
        for B in (S, Tw, D):
            assert np.array_equal(B.positions, pos)
        if f:
            seams += int(np.sum(want[:, 1] - kl.cpu().numpy()[want[:, 2]] + 1 < P))
        P += w
    assert seams > 2 * n                        # planted seams: keys across 256 and 257 overwrite each other in part


@pytest.mark.gpu
@pytest.mark.parametrize("w", [256, 272])
def test_eight_million_streams_one_and_two_segments(w):
    """2^23 streams of w-byte chunks: 2^31 bytes is one scan segment, 272 B makes two; a key across the boundary of
    every stream"""
    torch = _torch()
    keys, A = _c2()
    n = 1 << 23
    g = torch.Generator(device="cuda").manual_seed(w)
    text = _alnum(g, n, 2 * w)
    km, kl = _keymat(keys)
    _plant(text, w, km, kl, g)
    S = A.stream_batch(n)
    c = text[:, :w].contiguous()
    assert c.numel() == (1 << 31) * w // 256
    want0 = _arr(A.find_all_batch(c))
    assert np.array_equal(_arr(S.feed(c)), want0)
    c = text[:, w:].contiguous()
    got = _arr(S.feed(c))
    del c
    want = _new_part(_arr(A.find_all_batch(text)), np.full(n, w), np.arange(n))
    del text
    assert np.array_equal(got, want)
    assert len(want) > n
    assert np.array_equal(S.positions, np.full(n, 2 * w))


# ------------------------------------------------------------------ 2. long keys
LONG_ALPHA = {"bytes": [0x61, 0x62, 0x63, 0x64], "unicode": [0x61, 0x142, 0x1F600, 0x62]}


def _txt(kind, a):
    a = np.asarray(a)
    return a.astype(np.uint8).tobytes() if kind == "bytes" else a.astype("<u4").tobytes().decode("utf-32-le")


def _long_keys(kind, rng, longest):
    """keys cut from one random text, the longest `longest` letters, with prefixes and suffixes of each other; returns
    (keys, the text)"""
    base = rng.choice(LONG_ALPHA[kind], size=8 * longest)
    keys = {tuple(base[:longest].tolist())}
    for _ in range(10):
        ln = int(rng.integers(2, longest + 1))
        o = int(rng.integers(0, len(base) - ln + 1))
        keys.add(tuple(base[o:o + ln].tolist()))
    for k in sorted(keys):
        for _ in range(2):
            keys.add(k[:int(rng.integers(1, len(k) + 1))])
            keys.add(k[-int(rng.integers(1, len(k) + 1)):])
    return sorted(keys), base


def _windows(rng, base, n_streams, size):
    """each stream a window of `base` at a random offset (wrapping), a few letters changed"""
    src = []
    for _ in range(n_streams):
        x = np.take(base, int(rng.integers(0, len(base))) + np.arange(size), mode="wrap")
        flip = rng.integers(0, size, size=size // 500 + 1)
        x[flip] = rng.choice(base, size=len(flip))
        src.append(x)
    return src


def _plain_ragged(A, kind, hist, sel, before):
    """the plain scan of the histories of streams `sel` as (flat, offsets); the records past `before`"""
    batch = layout([hist[s] for s in sel], 1 if kind == "bytes" else 4)
    return _new_part(_arr(A.find_all_batch(batch)), before, np.asarray(sel))


def _long_key_streams(kind, keys, src, width, n_feeds, seed, gpu, long=False):
    """feed every stream its next chunk of width(s, f) letters of src[s]; ids: everyone on even feeds, a random half on
    odd ones.  Compared with the oracle per stream (long: the iter_long().set() chain) and, on the GPU, with the plain
    scan of whole streams; a twin batch gets every feed in two calls."""
    rng = np.random.default_rng(seed)
    A, O = automaton(kind, False, keys)
    n = len(src)
    S, Tw = A.stream_batch(n, long=long), A.stream_batch(n, long=long)
    hist = [s[:0] for s in src]
    its = [None] * n
    for f in range(n_feeds):
        ids = None if f % 2 == 0 else np.sort(rng.permutation(n)[:n // 2 + 1])
        sel = list(range(n)) if ids is None else ids.tolist()
        before = np.array([len(hist[s]) for s in sel], dtype=np.int64)
        chunks = [src[s][len(hist[s]):len(hist[s]) + width(s, f)] for s in sel]
        texts = [_txt(kind, c) for c in chunks]
        got = _arr(S.feed(texts, ids))
        want = []
        for s, c in zip(sel, chunks):
            hist[s] = np.concatenate([hist[s], c])
            if long:
                if its[s] is None:
                    its[s] = A.iter_long(_txt(kind, c))
                else:
                    its[s].set(_txt(kind, c))
                want += [(s, e, v) for e, v in its[s]]
            else:
                want += [(s, e, v) for e, v in O.find_all(_txt(kind, hist[s])) or [] if e >= len(hist[s]) - len(c)]
        want = np.array(want, dtype=np.int64).reshape(-1, 3)
        assert np.array_equal(got, want)
        if gpu and not long:
            assert np.array_equal(got, _plain_ragged(A, kind, hist, sel, before))
        assert np.array_equal(_split_feed(Tw, texts, ids, n), want)
        assert np.array_equal(Tw.positions, S.positions)
        assert S.positions.tolist() == [len(h) for h in hist]


def _long_case(kind, longest, n_streams, seed, gpu, long):
    rng = np.random.default_rng(seed)
    keys, base = _long_keys(kind, rng, longest)
    T = max(map(len, keys)) - 1
    assert T == longest - 1
    ws = [1, T - 1, T, T + 1, 3 * T]
    widths = rng.choice(ws, size=(n_streams, 5))
    src = _windows(rng, base, n_streams, int(widths.sum(axis=1).max()))
    _long_key_streams(kind, keys, src, lambda s, f: int(widths[s, f]), 5, seed, gpu, long)


@pytest.mark.gpu
@pytest.mark.parametrize("long", [False, True], ids=["find_all", "iter_long"])
@pytest.mark.parametrize("longest", [64, 1000, 5000])
@pytest.mark.parametrize("kind", ["bytes", "unicode"])
def test_long_keys_gpu(kind, longest, long):
    _long_case(kind, longest, 32, longest * 7 + len(kind), True, long)


def _runs_of_a(n_streams, n_feeds, seed, gpu, long):
    """a^1 ... a^64 and b a^63 (T = 63), stream s fed (s mod 70) + 1 letters a at a time, odd streams opened by b"""
    keys = [(0x61,) * i for i in range(1, 65)] + [(0x62,) + (0x61,) * 63]
    src = [np.array(([0x62] if s & 1 else []) + [0x61] * (70 * n_feeds), dtype=np.int64) for s in range(n_streams)]
    _long_key_streams("bytes", keys, src, lambda s, f: s % 70 + 1, n_feeds, seed, gpu, long)


@pytest.mark.gpu
@pytest.mark.parametrize("long", [False, True], ids=["find_all", "iter_long"])
def test_runs_of_one_letter_gpu(long):
    _runs_of_a(70, 3, 64, True, long)


@pytest.mark.parametrize("long", [False, True], ids=["find_all", "iter_long"])
def test_long_keys_emulated(long, monkeypatch):
    emul.install(monkeypatch)
    emul_streams.install(monkeypatch)
    _long_case("bytes", 64, 6, 9, False, long)
    _runs_of_a(5, 2, 10, False, long)


# ------------------------------------------------------------------ 3. tails past 2^31 bytes
@pytest.mark.gpu
def test_tails_past_2_31_bytes():
    """2^20 streams, a 2 100-letter key: T = 2 099, so the tails and the next-tail staging are 2.2 GB each.  Two feeds
    of 2 100-letter device chunks, a C2 key across every stream's boundary and the long key across every 64th
    stream's and the last 1 024 streams' (past the 2^31-byte mark of the tails)."""
    torch = _torch()
    keys, _ = _c2()
    g = torch.Generator(device="cuda").manual_seed(2100)
    long_key = bytes(_alnum(g, 1, 2100).cpu().numpy().reshape(-1))
    A = synth.build_automaton(keys + [long_key])
    n, w = 1 << 20, 2100
    assert n * (w - 1) > 2 ** 31
    text = _alnum(g, n, 2 * w)
    km, kl = _keymat(keys)
    _plant(text, w, km, kl, g)
    rows = torch.cat([torch.arange(0, n - 1024, 64, device="cuda"), torch.arange(n - 1024, n, device="cuda")])
    km, kl = _keymat([long_key])
    _plant(text, w, km, kl, g, rows)
    S = A.stream_batch(n)
    c = text[:, :w].contiguous()
    assert np.array_equal(_arr(S.feed(c)), _arr(A.find_all_batch(c)))
    c = text[:, w:].contiguous()
    got = _arr(S.feed(c))
    del c
    want = _new_part(_arr(A.find_all_batch(text)), np.full(n, w), np.arange(n))
    del text
    assert np.array_equal(got, want)
    lk = len(keys)
    assert int(np.sum(want[:, 2] == lk)) >= len(rows) and int(np.sum((want[:, 2] == lk) & (want[:, 0] >= n - 1024))) >= 1024
    assert np.array_equal(S.positions, np.full(n, 2 * w))


# ------------------------------------------------------------------ 4. iter_long batches at scale
@pytest.mark.gpu
def test_million_long_streams_equal_iter_long_chains():
    """2^20 long=True streams, three device feeds of 37, 5 and 64 letters over "abc": 500 sampled streams against the
    iter_long().set() chain, every stream against a twin fed in two calls"""
    torch = _torch()
    rng = np.random.default_rng(37)
    keys = sorted({tuple(rng.choice([0x61, 0x62, 0x63], size=int(rng.integers(3, 13))).tolist()) for _ in range(16)})
    A, _ = automaton("bytes", False, keys)
    n = 1 << 20
    S, Tw = A.stream_batch(n, long=True), A.stream_batch(n, long=True)
    g = torch.Generator(device="cuda").manual_seed(37)
    sample = np.sort(rng.permutation(n)[:500])
    its = {}
    for f, w in enumerate([37, 5, 64]):
        chunks = torch.randint(0, 3, (n, w), dtype=torch.uint8, device="cuda", generator=g) + 0x61
        got = _arr(S.feed(chunks))
        assert np.array_equal(_split_feed(Tw, chunks, None, n), got)
        host = chunks[torch.from_numpy(sample).cuda()].cpu().numpy()
        want = []
        for s, c in zip(sample.tolist(), host):
            c = c.tobytes()
            if f == 0:
                its[s] = A.iter_long(c)
            else:
                its[s].set(c)
            want += [(s, e, v) for e, v in its[s]]
        assert np.array_equal(got[np.isin(got[:, 0], sample)], np.array(want, dtype=np.int64).reshape(-1, 3))
        assert np.array_equal(S.positions, Tw.positions)
        assert np.array_equal(S.positions, np.full(n, [37, 42, 106][f]))


# ------------------------------------------------------------------ 5. shared table scratch
def _scratch_ops(rng):
    """(name, what it does to one automaton): stream batches fed from the host and the device, a pipelined
    find_all_batch, an iter_long(c0).set(c1) chain whose first chunk is handed over before the others run"""
    torch = _torch()
    keys = [bytes(rng.choice(np.frombuffer(b"abc", dtype=np.uint8), size=int(rng.integers(2, 10)))) for _ in range(30)]
    keys = sorted(set(keys))
    flat, off = _big_batch(rng, keys, 50 * MiB)
    feeds = [rng.choice(np.frombuffer(b"abc", dtype=np.uint8), size=(300, w)) for w in (5, 12, 3, 9)]
    c0, c1 = (bytes(rng.choice(np.frombuffer(b"abc", dtype=np.uint8), size=w)) for w in (4000, 900))
    state = {}

    def batch(A, long, k):
        key = ("long" if long else "all")
        if key not in state:
            state[key] = A.stream_batch(300, long=long)
        ids = None if k % 2 == 0 else np.arange(1, 300, 2)
        x = feeds[k] if ids is None else feeds[k][1::2].copy()
        if k in (1, 2):                                             # device feeds between host feeds
            x = torch.from_numpy(x).cuda()
        m = state[key].feed(x, ids)
        return _arr(m).tolist(), state[key].positions.tolist()

    def chain(A, step):
        if step == 0:
            state["it"] = A.iter_long(c0)
            return None
        if step == 1:
            r = list(state["it"])
            state["it"].set(c1)
            return r
        return list(state["it"])

    def big(A):
        return _arr(A.find_all_batch((flat, off))).tolist()

    ops = [("chain", lambda A: chain(A, 0))]
    for k in range(4):
        ops += [("all", lambda A, k=k: batch(A, False, k)), ("long", lambda A, k=k: batch(A, True, k))]
        if k == 1:
            ops += [("big", big), ("chain", lambda A: chain(A, 1))]
    ops += [("big", big), ("chain", lambda A: chain(A, 2))]
    return keys, ops, state, flat.size


@pytest.mark.gpu
def test_shared_table_scratch_keeps_every_user_apart():
    rng = np.random.default_rng(55)
    keys, ops, state, big_bytes = _scratch_ops(rng)
    assert big_bytes >= 48 * MiB                                    # the pipelined host route
    alone = {}
    for name in ("all", "long", "big", "chain"):
        A = synth.build_automaton(keys)
        state.clear()
        alone[name] = [f(A) for nm, f in ops if nm == name]
    A = synth.build_automaton(keys)
    state.clear()
    together = {name: [] for name in alone}
    for name, f in ops:
        together[name].append(f(A))
    for name in alone:
        assert together[name] == alone[name], name
    assert len(alone["big"][0]) > 8192 and alone["chain"][1] and alone["chain"][2]


# ------------------------------------------------------------------ 7. misaligned device views
@pytest.mark.gpu
@pytest.mark.parametrize("flavour", ["bytes", "unicode"])
def test_misaligned_device_views_equal_aligned_copies(flavour):
    """d[k:] of a [n, 7] (unicode: [n, 28]) uint8 CUDA tensor is contiguous but starts k*stride bytes into the
    storage: find_all_batch, find_long_batch and StreamBatch.feed take it as they take an aligned copy"""
    torch = _torch()
    rng = np.random.default_rng(16)
    keys = sorted({bytes(rng.choice(np.frombuffer(b"abc", dtype=np.uint8), size=int(rng.integers(2, 9)))) for _ in range(20)})
    mod = pkg.flavour(flavour)
    A = mod.Automaton(mod.STORE_INTS)
    for i, k in enumerate(keys):
        A.add_word(k if flavour == "bytes" else k.decode(), i)
    A.make_automaton()
    L = 1 if flavour == "bytes" else 4
    rows = rng.choice(np.frombuffer(b"abc", dtype=np.uint8), size=(400, 7)).astype(np.dtype(f"<u{L}"))
    d = torch.from_numpy(rows.view(np.uint8).copy()).cuda()
    for k in (1, 3, 5):
        v = d[k:]
        assert v.is_contiguous() and v.data_ptr() % 16
        c = v.clone()
        for run in (A.find_all_batch, A.find_long_batch):
            got, want = run(v), run(c)
            assert len(want) > 100 and np.array_equal(_arr(got), _arr(want))
        Sv, Sc = A.stream_batch(400), A.stream_batch(400)
        for _ in range(2):
            assert np.array_equal(_arr(Sv.feed(v)), _arr(Sc.feed(c)))
        assert np.array_equal(Sv.positions, Sc.positions)


@pytest.mark.gpu
def test_c_abi_still_refuses_misaligned_buffers():
    """the C entries keep their check: a device pointer off a 16-byte boundary is ACB_EINVAL"""
    torch = _torch()
    A, _ = automaton("bytes", False, [tuple(b"ab")])
    lib, tb = A._lib, A._ensure_table(0)
    d = torch.zeros(64, dtype=torch.uint8, device="cuda")
    cnt = torch.zeros(1, dtype=torch.int64, device="cuda")
    out = torch.zeros((16, 3), dtype=torch.int32, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    assert lib.acb_scan_device(tb, d.data_ptr() + 1, 7, None, 1, 7, out.data_ptr(), 16, cnt.data_ptr(), s, 0) == N.ACB_EINVAL
    ss = ctypes.c_void_p()
    N.check(lib.acb_streams_new(tb, 1, 0, ctypes.byref(ss)))
    try:
        assert lib.acb_streams_feed_device(ss, tb, d.data_ptr() + 8, 7, None, 1, 7, None, out.data_ptr(), 16,
                                           cnt.data_ptr(), s, 0) == N.ACB_EINVAL
    finally:
        lib.acb_streams_free(ss)
