"""find_all_batch(..., ignore_white_space=True) and stream_batch(..., ignore_white_space=True): white space removed on
the GPU before the scan, records mapped back to original letters.

The answer is always the reference's iter(hay, ignore_white_space=True) -- the C oracle's, whose letters widen bytes
like the reference -- or its iter(c0, ignore_white_space=True) ... .set(c1) chain for streams; at scale, a plain
find_all_batch of the batch with the white space cut out, mapped back through the kept columns.  Every randomised test
has a CPU form on the numpy restatement (tests/emul_white_space.py) and a gpu-marked twin on the real kernels."""
import ctypes

import numpy as np
import pytest

import emul_white_space
from batch_cases import automaton, fake_table, forms, got_values, obj, table_and_batch, triples
from pyahocorasick_b200 import _native as N
from pyahocorasick_b200 import automaton as am

WS = [0x20, 0x09, 0x0A, 0x0B, 0x0C, 0x0D, 0x85, 0xA0, 0x1C, 0x1D, 0x1E, 0x1F]
WIDE_WS = list(range(0x2000, 0x200B)) + [0x2028, 0x2029, 0x3000]

_libc = ctypes.CDLL(None)
_libc.iswspace.argtypes = [ctypes.c_uint]
_libc.iswspace.restype = ctypes.c_int


def _space_letters(L, signed):
    n = ctypes.c_int64(0)
    out = np.empty(4096, dtype=np.uint32)
    assert N.lib().acb_space_letters(L, signed, N.ptr(out), len(out), ctypes.byref(n)) == N.ACB_OK
    return out[:n.value].tolist()


# ------------------------------------------------------------------ the predicate
@pytest.mark.parametrize("signed", [0, 1])
def test_space_letters_of_bytes_equal_libc(signed):
    want = [b for b in range(256) if _libc.iswspace((b - 256) & 0xFFFF if signed and b >= 128 else b)]
    assert _space_letters(1, signed) == want


def test_space_letters_of_2_and_4_byte_letters_equal_libc():
    assert _space_letters(2, 0) == [v for v in range(1 << 16) if _libc.iswspace(v)]
    assert _space_letters(4, 0) == [v for v in range(0x110000) if _libc.iswspace(v)]
    rng = np.random.default_rng(0)
    assert not any(_libc.iswspace(int(v)) for v in rng.integers(0x110000, 1 << 32, size=20000))


def test_space_letters_report_the_size_on_overflow():
    n = ctypes.c_int64(0)
    out = np.empty(1, dtype=np.uint32)
    assert N.lib().acb_space_letters(4, 0, N.ptr(out), 1, ctypes.byref(n)) == N.ACB_EOVERFLOW
    assert n.value == len(_space_letters(4, 0)) > 1
    assert N.lib().acb_space_letters(3, 0, N.ptr(out), 1, ctypes.byref(n)) == N.ACB_EINVAL


def test_space_mask_takes_the_same_set():
    """iter()'s host compaction and the batch scans share one definition of white space"""
    b = np.arange(256, dtype=np.uint8)
    assert np.nonzero(am._space_mask(b, True))[0].tolist() == _space_letters(1, 1)
    assert np.nonzero(am._space_mask(b, False))[0].tolist() == _space_letters(1, 0)
    w = np.arange(0x110000, dtype=np.uint32)
    assert np.nonzero(am._space_mask(w, False))[0].tolist() == _space_letters(4, 0)


# ------------------------------------------------------------------ argument errors
def test_skip_argument_errors():
    L = N.lib()
    fake = ctypes.addressof(fake_table())                       # never used as a table: the skip set is checked first
    n = ctypes.c_int64(0)
    ok = np.array([9, 32], dtype=np.uint32)
    bad = np.array([32, 9], dtype=np.uint32)
    dup = np.array([9, 9], dtype=np.uint32)
    big = np.arange(N.MAX_SKIP + 1, dtype=np.uint32)
    hay = np.zeros(16, dtype=np.uint8)
    for skip, algo in ((ok, N.ALGO_LONG), (bad, N.ALGO_AUTO), (dup, N.ALGO_FILTER), (big, N.ALGO_DFA)):
        assert L.acb_scan_host_skip(fake, N.ptr(hay), 16, None, 1, 16, None, 8, ctypes.byref(n), algo, 1, N.ptr(skip), len(skip)) == N.ACB_EINVAL
        assert L.acb_scan_device_skip(fake, N.ptr(hay), 16, None, 1, 16, None, 0, N.ptr(hay), None, algo, N.ptr(skip), len(skip)) == N.ACB_EINVAL
    for skip in (bad, dup, big):
        ss = ctypes.c_void_p()
        assert L.acb_streams_new_skip(fake, 4, N.ptr(skip), len(skip), ctypes.byref(ss)) == N.ACB_EINVAL and not ss.value
    A = automaton("bytes", False, [b"ab"])[0]
    with pytest.raises(ValueError):
        A.find_all_batch([b"a b"], algo="long", ignore_white_space=True)
    with pytest.raises(ValueError):
        A.stream_batch(3, long=True, ignore_white_space=True)


# ------------------------------------------------------------------ batches against the oracle
def _want(O, hays):
    return [(h, e, v) for h, hay in enumerate(hays) for e, v in O.iter(hay, ignore_white_space=True)]


# (flavour, key type, alphabet of text letters) -- latin-1, wide and mixed unicode; bytes-flavour sequences are
# 2-byte letters, unicode-flavour sequences 4-byte ones
CASES = {
    "bytes": ("bytes", False, [0x61, 0x62, 0xE9] + WS),
    "latin1": ("unicode", False, [0x61, 0x62, 0xE9] + WS),
    "wide": ("unicode", False, [0x61, 0x142, 0x1F600] + WS + WIDE_WS),
    "mixed": ("unicode", False, [0x61, 0x62] + WS + WIDE_WS),
    "seq2": ("bytes", True, [0x61, 0x6162, 0xFF20] + WS + WIDE_WS),
    "seq4": ("unicode", True, [0x61, 0x1F600, 0x10FFFF] + WS + WIDE_WS),
}


def _random_case(case, rng):
    fl, seq, al = CASES[case]
    words = [0x61, 0x62] if case in ("bytes", "latin1", "mixed") else al[:3]
    keys = {tuple(int(x) for x in rng.choice(words, size=int(rng.integers(1, 6)))) for _ in range(int(rng.integers(1, 8)))}
    keys |= {tuple(int(x) for x in rng.choice(al, size=int(rng.integers(1, 4)))) for _ in range(2)}   # keys with white space
    A, O = automaton(fl, seq, sorted(keys))
    n = int(rng.integers(1, 12))
    hays = []
    for _ in range(n):
        r = int(rng.integers(0, 5))
        if r == 0:
            hays.append([])
        elif r == 1:
            hays.append([int(x) for x in rng.choice(WS, size=int(rng.integers(1, 9)))])     # all white space
        else:
            hays.append([int(x) for x in rng.choice(al, size=int(rng.integers(0, 60)))])
    if case == "mixed" and all(max(h, default=0) < 256 for h in hays):
        hays.append([0x1F600, 0x20, 0x61])
    return A, O, hays


def _batches(cases, seed, trials, algo="auto", sort=True):
    rng = np.random.default_rng(seed)
    for case in cases:
        for _ in range(trials):
            A, O, hays = _random_case(case, rng)
            if rng.integers(0, 3) == 0:                           # a fixed-stride batch too
                w = int(rng.integers(1, 20))
                hays = [(h + [0x61] * w)[:w] for h in hays]
            objs = [obj(*CASES[case][:2], h) for h in hays]
            want = _want(O, objs)
            for form, x in forms(objs, hays, A._L, case in ("latin1", "mixed")):
                got = triples(A.find_all_batch(x, algo=algo, sort=sort, ignore_white_space=True))
                if not sort:
                    got, want_ = sorted(got), sorted(want)
                else:
                    want_ = want
                assert got == want_, (case, form, hays)


@pytest.mark.parametrize("case", list(CASES))
def test_batches_match_oracle_emulated(case, monkeypatch):
    emul_white_space.install(monkeypatch)
    _batches([case], 7, 25)


@pytest.mark.gpu
@pytest.mark.parametrize("algo", ["filter", "dfa"])
@pytest.mark.parametrize("case", list(CASES))
def test_batches_match_oracle_gpu(case, algo):
    _batches([case], 107, 40, algo=algo)
    _batches([case], 207, 10, algo=algo, sort=False)


def test_batches_equal_the_drop_in_iter(monkeypatch):
    """the drop-in's own iter(..., ignore_white_space=True) (host compaction) gives the same records"""
    emul_white_space.install(monkeypatch)
    rng = np.random.default_rng(3)
    for case in CASES:
        A, O, hays = _random_case(case, rng)
        objs = [obj(*CASES[case][:2], h) for h in hays]
        want = [(h, e, v) for h, o in enumerate(objs) for e, v in A.iter(o, ignore_white_space=True)]
        assert got_values(A.find_all_batch(objs, ignore_white_space=True)) == want


# ------------------------------------------------------------------ streams against the oracle's iter().set() chain
STREAM_CASES = ["bytes", "seq2", "seq4", "wide"]


def _streams(case, seed, n_streams, n_feeds, algo="auto"):
    rng = np.random.default_rng(seed)
    fl, seq, al = CASES[case]
    A, O, _ = _random_case(case, rng)
    S = A.stream_batch(n_streams, algo=algo, ignore_white_space=True)
    its, pos = [None] * n_streams, [0] * n_streams
    T = max(A.get_stats()["longest_word"] - 1, 1)
    for f in range(n_feeds):
        if f == n_feeds // 2:
            gone = rng.permutation(n_streams)[:n_streams // 3]
            S.reset(gone)
            for s in gone.tolist():
                its[s], pos[s] = None, 0
        ids = rng.permutation(n_streams)[:int(rng.integers(1, n_streams + 1))]
        chunks = []
        for _ in ids:
            r = int(rng.integers(0, 4))
            n = [0, int(rng.integers(0, T + 1)), int(rng.integers(0, 3 * T + 4)), 30][r]
            pool = WS if rng.integers(0, 4) == 0 else al                  # chunks of white space only
            chunks.append([int(x) for x in rng.choice(pool, size=n)])
        m = S.feed([obj(fl, seq, c) for c in chunks], ids)
        want = []
        for s, c in sorted(zip(ids.tolist(), chunks), key=lambda x: x[0]):
            if its[s] is None:
                its[s] = O.iter(obj(fl, seq, c), ignore_white_space=True)
            else:
                its[s].set(obj(fl, seq, c))
            want += [(s, e, v) for e, v in its[s]]
            pos[s] += len(c)
        order = {s: i for i, s in enumerate(ids.tolist())}
        want.sort(key=lambda r: order[r[0]])                              # records come in chunk order
        got = triples(m)
        assert sorted(got) == sorted(want) and [r[0] for r in got] == [r[0] for r in want], (case, f)
        assert S.positions.tolist() == pos


@pytest.mark.parametrize("case", STREAM_CASES)
def test_streams_match_oracle_chain_emulated(case, monkeypatch):
    emul_white_space.install(monkeypatch)
    _streams(case, 13, 9, 8)


@pytest.mark.gpu
@pytest.mark.parametrize("algo", ["filter", "dfa"])
@pytest.mark.parametrize("case", STREAM_CASES)
def test_streams_match_oracle_chain_gpu(case, algo):
    _streams(case, 113, 200, 8, algo)


# ------------------------------------------------------------------ GPU: overflow, boundaries, scale, device tensors
@pytest.mark.gpu
def test_overflow_counts_exactly_and_stream_feeds_commit_nothing():
    rng = np.random.default_rng(1)
    A, O = automaton("bytes", False, [b"ab", b"abc", b"b", b"ca"])
    hays = [bytes(rng.choice(list(b"abc \t"), size=40).tolist()) for _ in range(30)]
    want = _want(O, hays)
    n = len(want)
    skip = A._skip_set(False)
    tb, flat, offs = table_and_batch(A, hays)
    lib = N.lib()
    for cap in (0, 1, n - 1):
        found = ctypes.c_int64(0)
        out = np.empty(max(cap, 1), dtype=N.MATCH_DTYPE)
        rc = lib.acb_scan_host_skip(tb, N.ptr(flat), flat.size, N.ptr(offs), len(hays), 0, N.ptr(out), cap, ctypes.byref(found),
                                    N.ALGO_FILTER, 1, N.ptr(skip), len(skip))
        assert rc == N.ACB_EOVERFLOW and found.value == n
    import torch
    d = torch.from_numpy(flat.copy()).cuda()
    do = torch.from_numpy(offs).cuda()
    cnt = torch.zeros(1, dtype=torch.int64, device="cuda")
    for cap in (0, 1, n - 1):
        out = torch.empty((max(cap, 1), 3), dtype=torch.int32, device="cuda")
        N.check(lib.acb_scan_device_skip(tb, d.data_ptr(), flat.size, do.data_ptr(), len(hays), 0, out.data_ptr(), cap,
                                         cnt.data_ptr(), None, N.ALGO_DFA, N.ptr(skip), len(skip)))
        torch.cuda.synchronize()
        assert int(cnt.item()) == n
        stored = {tuple(r) for r in out[:cap].cpu().tolist()}
        assert stored <= set(want)                             # stored records are mapped back
    S = A.stream_batch(len(hays), ignore_white_space=True)
    first = S.feed(hays)
    assert triples(first) == want
    second = [h[::-1] for h in hays]
    its = [O.iter(h, ignore_white_space=True) for h in hays]
    want2 = []
    for s, it in enumerate(its):
        list(it)
        it.set(second[s])
        want2 += [(s, e, v) for e, v in it]
    ss, before = S._ss, S.positions.copy()
    found = ctypes.c_int64(0)
    f2 = np.frombuffer(b"".join(second), dtype=np.uint8)
    rc = lib.acb_streams_feed_host(ss, tb, N.ptr(f2), f2.size, N.ptr(offs), len(hays), 0, None, None, 1, ctypes.byref(found), N.ALGO_FILTER, 1)
    assert rc == N.ACB_EOVERFLOW and found.value == len(want2) and (S.positions == before).all()
    assert triples(S.feed(second)) == want2                  # the same feed again, with room
    assert S.positions.tolist() == [2 * len(h) for h in hays]


# letter width -> (flavour, key sequences?, text letters, key, white-space letters): the 2- and 4-byte cases hold letters
# outside latin-1, so that they run at their own width and never on the latin-1 table
WIDTHS = {
    1: ("bytes", False, [0x61, 0x62, 0x63, 0x64], list(b"qrstuvwx"), [0x20, 0x09, 0x0A]),
    2: ("bytes", True, [0x61, 0x6162, 0x142, 0x63], [0x71, 0x72, 0x142, 0x74, 0x75, 0x6162, 0x77, 0x78], [0x20, 0x3000, 0x2028]),
    4: ("unicode", False, [0x61, 0x142, 0x1F600, 0x63], [0x71, 0x72, 0x142, 0x74, 0x75, 0x1F600, 0x77, 0x78], [0x20, 0x3000, 0x2028, 0x0A]),
}


def _boundary_text(L, rng):
    """letters of one haystack with the key planted, split by a white-space run, across
    A) the scan's 1 KiB slice, 20 and 32 KiB tile and 16-byte run boundaries at every letter-aligned residue -- placed in
       the COMPACTED text, which is what the scan sees -- and
    B) the compaction's 8 192-letter tile boundaries of the ORIGINAL text (a white-space pad moves the split onto the
       next one).
    Returns (letters, number of planted keys, tile boundaries straddled by a run inside a key)."""
    _, _, base, key, ws = WIDTHS[L]
    n = 20 * 8192 + 77
    C = [int(x) for x in rng.choice(base, size=n)]
    byte_cuts = [(3 + 4 * r) * 1024 + r * L for r in range(16 // L)] + [20480 * k + L for k in (1, 3, 7)] + [32768 * k for k in (1, 2, 3)]
    plants, used = {}, []                                      # compacted start of a key -> ("A" | "B", split)

    def free(q):
        return q + len(key) < n and all(abs(q - u) > 64 for u in used)
    for i, bc in enumerate(byte_cuts):
        c = bc // L                                             # a letter boundary of the compacted text
        j = 1 + i % (len(key) - 1)
        assert free(c - j)
        plants[c - j] = ("A", j)
        used.append(c - j)
    for q in range(3000, n - 100, 5000):
        while not free(q):
            q += 97
        plants[q] = ("B", 1 + (q // 5000) % (len(key) - 1))
        used.append(q)
    for q in plants:
        C[q:q + len(key)] = key
    out, straddled, i = [], set(), 0
    for q in sorted(plants):
        out += C[i:q]
        kind, j = plants[q]
        run = 1 + (q % 37)
        if kind == "B":                                         # pad so that the run inside the key straddles a tile boundary
            tile = -(-(len(out) + j + run // 2) // 8192) * 8192
            out += [ws[x % len(ws)] for x in range(tile - run // 2 - len(out) - j)]
            straddled.add(tile)
        out += key[:j] + [ws[x % len(ws)] for x in range(run)] + key[j:]
        i = q + len(key)
    out += C[i:]
    return out, len(plants), straddled


@pytest.mark.gpu
@pytest.mark.parametrize("L", [1, 2, 4])
def test_white_space_runs_and_keys_across_every_boundary(L):
    """keys split by white space across every compaction-tile boundary and every scan boundary, at 1-, 2- and 4-byte
    letters; several tiles each, so the look-back, later tiles' prefixes, unaligned stores and the remap's search over
    tiles all run at every width"""
    fl, seq, _, key, ws = WIDTHS[L]
    A, O = automaton(fl, seq, [key, [0x7A, 0x7A]])
    assert A._L == L
    letters, n_plants, straddled = _boundary_text(L, np.random.default_rng(L))
    assert len(straddled) >= 15 and len(letters) > 20 * 8192
    objs = [obj(fl, seq, letters), obj(fl, seq, letters[1:]), obj(fl, seq, letters[:8191] + ws[:1] * 2 + letters[8191:])]
    batch = A._batch_input(objs)
    assert batch[0] == "host" and batch[5] is False and batch[1].size == L * sum(len(o) for o in objs)   # not the latin-1 table
    want = _want(O, objs)
    assert sum(1 for r in want if r[2] == 0) >= 3 * n_plants - 1
    for algo in ("filter", "dfa"):
        assert triples(A.find_all_batch(objs, algo=algo, ignore_white_space=True)) == want


def _column_reference(A, x, keep_cols, algo="auto"):
    """records of a plain find_all_batch over x[:, keep_cols], end_index mapped back through keep_cols"""
    import torch
    m = A.find_all_batch(x[:, keep_cols].contiguous(), algo=algo)
    return list(zip(m.hay_id.tolist(), keep_cols.cpu().numpy()[m.end_index].tolist(), m.key_id.tolist()))


@pytest.mark.gpu
def test_batch_without_white_space_is_byte_identical():
    from pyahocorasick_b200 import synth
    w = synth.make("C2", scale=0.05)
    A = synth.build_automaton(w.keys)
    x = w.haystacks.copy()
    x[np.isin(x, np.array(A._skip_set(False), dtype=np.uint8))] = ord("x")
    for algo in ("filter", "dfa"):
        a = A.find_all_batch(x, algo=algo)
        b = A.find_all_batch(x, algo=algo, ignore_white_space=True)
        assert np.array_equal(np.asarray(a.hay_id), np.asarray(b.hay_id)) and np.array_equal(a.end_index, b.end_index) \
            and np.array_equal(a.key_id, b.key_id)


def _scale(n, stride, seed, host=True):
    """C2 keys, white space at fixed columns (every 13th, from a random phase) so that the reference is a plain scan of
    the kept columns; the compaction itself sees a flat buffer whose runs fall anywhere relative to its tiles"""
    import torch
    from pyahocorasick_b200 import synth
    w = synth.make("C2", scale=0.01)
    A = synth.build_automaton(w.keys)
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randint(ord("a"), ord("z") + 1, (n, stride), dtype=torch.uint8, device="cuda", generator=g)
    for i, k in enumerate(w.keys[:64]):                         # planted keys
        kk = torch.tensor(list(k), dtype=torch.uint8, device="cuda")
        x[i * (n // 64), 40:40 + len(k)] = kk
    cols = torch.arange(stride, device="cuda")
    ws = (cols % 13) == 5
    x[:, ws] = ord(" ")
    want = _column_reference(A, x, cols[~ws])
    m = A.find_all_batch(x.cpu().numpy() if host else x, ignore_white_space=True)
    assert triples(m) == want
    return len(want)


@pytest.mark.gpu
def test_48_mib_batch():
    assert _scale(49152, 1024 + 17, 5) > 0


@pytest.mark.gpu
def test_batch_past_2_31_bytes_and_two_compacted_segments():
    """2^31 + 2^28 bytes; 12 of every 13 columns are kept, so the compacted batch is past 2 GiB as well"""
    assert _scale(1 << 21, 1152, 6, host=False) > 0


@pytest.mark.gpu
def test_device_tensors_and_a_misaligned_view():
    import torch
    rng = np.random.default_rng(8)
    A, O = automaton("bytes", False, [b"ab", b"b c", b"ca", b"abcab"])
    x = rng.choice(np.frombuffer(b"abc \t\x85", dtype=np.uint8), size=(301, 7))
    want = _want(O, [bytes(r) for r in x])
    d = torch.from_numpy(x).cuda()
    assert triples(A.find_all_batch(d, ignore_white_space=True)) == want
    v = d[1:]
    assert v.data_ptr() % 16
    assert triples(A.find_all_batch(v, ignore_white_space=True)) == [(h - 1, e, k) for h, e, k in want if h]


@pytest.mark.gpu
def test_two_to_the_20_streams_with_white_space_at_the_seams():
    import torch
    from pyahocorasick_b200 import synth
    w = synth.make("C2", scale=0.01)
    A = synth.build_automaton(w.keys)
    n = 1 << 20
    key = max(w.keys[:200], key=len)
    kid = w.keys.index(key)
    S = A.stream_batch(n, ignore_white_space=True)
    j = np.arange(n) % (len(key) - 1) + 1                     # split point of the key in stream s
    r = np.arange(n) % 5                                      # white space before the seam
    c0 = np.full((n, 64), ord("#"), dtype=np.uint8)
    c1 = np.full((n, 64), ord("#"), dtype=np.uint8)
    kb = np.frombuffer(key, dtype=np.uint8)
    for jj in range(1, len(key)):
        for rr in range(5):
            sel = (j == jj) & (r == rr)
            c0[sel, 64 - jj - rr:64 - rr] = kb[:jj]
            c0[sel, 64 - rr:] = ord(" ")
            c1[sel, :3] = ord("\t")
            c1[sel, 3:3 + len(key) - jj] = kb[jj:]
    S.feed(torch.from_numpy(c0).cuda())
    m = S.feed(torch.from_numpy(c1).cuda())
    got = np.asarray(m.key_id) == kid
    assert got.sum() == n
    assert (np.asarray(m.hay_id)[got] == np.arange(n)).all()
    assert (np.asarray(m.end_index)[got] == 64 + 3 + len(key) - j - 1).all()
    assert (S.positions == 128).all()
