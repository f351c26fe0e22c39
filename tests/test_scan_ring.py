"""The scan kernels' tile rings through many turns per CTA, against the C oracle.

Both filter scan kernels are persistent: one CTA per SM, a producer warp that claims tiles from a global counter
(claim_depth claims in flight) and loads them into a ring of `stages` shared-memory stages guarded by mbarriers; fill f
uses stage f % stages with the barrier parity (f / stages) & 1, sentinel fills end the consumers, and the last CTA to
finish re-arms the counter for the next launch.  Most of what can go wrong there (a parity, a stale look-ahead or zero
fill in a reused stage, pair-kernel candidates held across a released stage, a sentinel at an unusual ring phase, a
counter left armed) shows only once a CTA has used a stage more than once -- and on a 132-SM H100 a text of a few tiles
gives each CTA one or two fills, in an order decided by the race of the claims.

acb_table_set_cta_limit makes a table launch as if the device had fewer SMs, so at limit 1 tile f is fill f of the one
CTA; acb_table_scan_grid reports the launch shape the scans compute, so every test asserts the shape it meant to get;
acb_scan_geometry reports each kernel's ring, so the texts follow the build (tile size, stages, claim depth):

  CPU    the geometry against the invariants the kernels rely on, and the tile kernel_cells plants at.
  GPU    ring turnover at limit 1 on one cell per kernel instantiation (6 * stages + 1 tiles, dense windows on each
         stage's first reuse in both parities, candidates held past a released stage), then at limits 2, 3 and 0;
         the end of work at every ring phase (tile counts around the stages and the claim depth, last tiles of every
         copy shape) with a scan at other limits after each; the full grid at about 32 MiB; and the grid-stride loops
         of the batch features (selection, word filter, replacement, white-space remap, stream gather) at one SM.
"""
import ctypes
import re

import numpy as np
import pytest

import emul_leftmost
import emul_replace
import emul_words
import pyahocorasick_b200 as ac
from pyahocorasick_b200 import _native as N
from batch_cases import CASES, DT, automaton, obj, oracle_full, rows
from kernel_cells import (ALPHA, CELLS, SLICE, Cell, _build, _check_shape, _dense, _diff, _keys, _oracle, _ragged, _seed,
                          _text, _want, all_instantiations, cell_instantiation, geometry, sentinels, tile_bytes)

SPARSE = 0x23                     # '#': a letter of no key in any cell


# ------------------------------------------------------------------ the hooks
@pytest.fixture
def cta_limit():
    """limit(A, n): the CTA limit of A's device-0 tables (and its latin-1 one); every table is set back to 0 after"""
    seen = []

    def limit(A, n):
        tbs = [A._ensure_table(0)]
        if A._UNICODE and A._key_type != ac.KEY_SEQUENCE:            # key sequences have no latin-1 automaton
            core = A._ensure_narrow(0)
            if core is not None:
                tbs.append(core[1])
        for tb in tbs:
            N.check(N.lib().acb_table_set_cta_limit(tb, n))
            seen.append((A, tb))
    yield limit
    for _, tb in seen:
        N.check(N.lib().acb_table_set_cta_limit(tb, 0))


def scan_grid(A, total_bytes):
    """(CTAs, tiles) of a filter scan of total_bytes on A's device-0 table"""
    grid, tiles = ctypes.c_int32(), ctypes.c_int64()
    N.check(N.lib().acb_table_scan_grid(A._ensure_table(0), int(total_bytes), ctypes.byref(grid), ctypes.byref(tiles)))
    return grid.value, tiles.value


# ------------------------------------------------------------------ CPU: the geometry
@pytest.mark.parametrize("pair", [False, True], ids=["stream", "pair"])
def test_scan_geometry_invariants(pair):
    r = geometry(pair)
    slices = r.tile // r.slice
    assert r.slice == SLICE == 1024 and r.tile == slices * r.slice and r.tile % 16 == 0
    assert r.stages >= 2 and r.claim_depth >= 1 and r.look >= 16 and r.consumers >= 1
    assert sentinels(r) <= r.stages                                 # sentinel fills never wrap the ring
    assert (r.consumers + slices - 1) // slices + 2 < 2 * r.stages   # the fills in use never alias a barrier phase
    if pair:
        assert slices & (slices - 1) == 0 and r.stages & (r.stages - 1) == 0     # split by shifts and masks


def test_scan_geometry_refuses_a_short_buffer():
    out = (ctypes.c_int32 * 6)(*[-1] * 6)
    assert N.lib().acb_scan_geometry(0, out, 5) == N.ACB_EINVAL and list(out) == [-1] * 6
    assert N.lib().acb_scan_geometry(1, None, 6) == N.ACB_EINVAL
    assert N.lib().acb_table_set_cta_limit(None, 1) == N.ACB_EINVAL
    assert N.lib().acb_table_scan_grid(None, 1, ctypes.byref(ctypes.c_int32()), ctypes.byref(ctypes.c_int64())) == N.ACB_EINVAL


@pytest.mark.parametrize("cell", CELLS, ids=[c.name for c in CELLS])
def test_cells_plant_at_the_tiles_of_their_kernel(cell):
    """the kernel matrix and the record-bound tests plant at the tile of the kernel a cell runs, as the library reports
    it: _text's last three boundary plants (the tile-level ones; the text has room for all three) start just before
    1, 2 and 3 tiles"""
    tile = geometry(cell.pair).tile
    assert tile_bytes(cell) == tile
    rng = np.random.Generator(np.random.PCG64(_seed(cell)))
    keys = _keys(cell, rng)
    assert max(map(len, keys)) * cell.L < 256
    _, starts = _text(cell, keys, rng, 3 * tile + 4 * SLICE)
    at = starts[-3:] * cell.L
    assert all(j * tile - 256 < a < j * tile for j, a in zip((1, 2, 3), at)), (tile, at.tolist())


# ------------------------------------------------------------------ comparing records
def _rows_of(want):
    return np.asarray(want, dtype=np.int64).reshape(-1, 3)


def _keyed(r):
    """records as one sortable int64 each, for comparing an unsorted result as a multiset"""
    assert r[:, 0].max(initial=0) < 1 << 23 and r[:, 1].max(initial=0) < 1 << 25 and r[:, 2].max(initial=0) < 1 << 15
    return np.sort((r[:, 0] << 40) | (r[:, 1] << 15) | r[:, 2])


def _same(got, want, what):
    if not np.array_equal(got, want):
        pytest.fail(f"{what}: {_diff([tuple(x) for x in got.tolist()], [tuple(x) for x in want.tolist()])}")


def _check_scan(A, batch, want, what, dfa=False):
    _same(rows(A.find_all_batch(batch, algo="filter")), want, f"{what}, filter")
    if not np.array_equal(_keyed(rows(A.find_all_batch(batch, algo="filter", sort=False))), _keyed(want)):
        pytest.fail(f"{what}, filter unsorted: not the oracle's records")
    if dfa:
        _same(rows(A.find_all_batch(batch, algo="dfa")), want, f"{what}, dfa")


# ------------------------------------------------------------------ GPU: ring turnover in one CTA
def _ring_cells():
    """one stream cell per instantiation (letter widths rotating where the instantiation allows more than one), the
    pair kernel at every level-1 size and with the tag bitmap"""
    by = {}
    for c in CELLS:
        if not (c.pair or c.log1 or c.tagmap):
            by.setdefault(cell_instantiation(c), []).append(c)
    stream = [cs[i % len(cs)] for i, (_, cs) in enumerate(sorted(by.items(), key=str))]
    pair = [c for c in CELLS if c.pair and not c.tagmap] + [next(c for c in CELLS if c.pair and c.tagmap)]
    return stream + pair


RING_CELLS = _ring_cells()


def _alternate(cell, n):
    x, y = ALPHA[cell.L][:2]
    return np.resize(np.array([x, y], dtype=np.uint32), n)


def _ring_text(cell, keys, rng, ring):
    """6 * stages + 1 tiles and a ragged tail: _text's boundary plants; dense windows of 3 slices across the tile
    boundaries around fills S, S + 1 and 2S (each stage's first reuse, in both parities); a dense window that ends 5
    letters before a tile boundary, followed by a sparse tile (candidates still held when their stage is released)"""
    L, S = cell.L, ring.stages
    tl, sl = ring.tile // L, SLICE // L
    t, starts = _text(cell, keys, rng, (6 * S + 1) * ring.tile + 3000 + L * 1291)
    for f in (S, S + 1, 2 * S):
        for b in (f * tl, (f + 1) * tl):
            t[b - 3 * sl // 2:b + 3 * sl // 2] = _alternate(cell, 3 * sl)
    b = (4 * S + 1) * tl
    t[b - 3 * sl - 5:b - 5] = _alternate(cell, 3 * sl)
    t[b - 5:b + tl] = SPARSE
    plant = [k for k in keys if len(k) >= 2]
    for i, p in enumerate(range(b + 7, b + tl - 64, 4096 // L)):
        k = plant[i % len(plant)]
        t[p:p + len(k)] = k
    return t, starts


@pytest.mark.gpu
@pytest.mark.parametrize("cell", RING_CELLS, ids=[c.name for c in RING_CELLS])
def test_ring_turns_over_in_one_cta(cell, monkeypatch, cta_limit):
    rng = np.random.Generator(np.random.PCG64(_seed(cell) + 1))
    keys = _keys(cell, rng)
    A = _build(cell, keys, monkeypatch)
    _check_shape(A, cell)
    O = _oracle(cell, keys)
    ring = geometry(cell.pair)
    L, dt, S = cell.L, DT[cell.L], ring.stages
    t, starts = _ring_text(cell, keys, rng, ring)
    n = t.size
    flat = t.astype(dt).view(np.uint8)
    tl = ring.tile // L
    layouts = [("one haystack", (flat, np.array([0, n], dtype=np.int64) * L), t, np.array([0, n], dtype=np.int64))]
    roff = _ragged(rng, n, starts, np.repeat(np.arange(tl, n, tl), 3))            # runs of empty haystacks on every boundary
    layouts.append(("ragged batch", (flat, roff * L), t, roff))
    for stride in (512, 3000):
        k = flat.size // stride
        layouts.append((f"stride {stride}", flat[:k * stride].reshape(k, stride), t[:k * (stride // L)],
                        np.arange(k + 1, dtype=np.int64) * (stride // L)))
    d = _dense(cell, (6 * S + 1) * ring.tile + L * 1291)
    layouts.append(("dense text", (d.astype(dt).view(np.uint8), np.array([0, d.size * L], dtype=np.int64)), d,
                    np.array([0, d.size], dtype=np.int64)))
    for what, batch, letters, off in layouts:
        want = _rows_of(_want(O, cell, letters, off))
        total = int(off[-1]) * L
        cta_limit(A, 1)
        grid, tiles = scan_grid(A, total)
        assert grid == 1 and tiles >= 6 * S + 1, (what, grid, tiles)
        _check_scan(A, batch, want, f"{what}, limit 1", dfa=True)
        if what in ("one haystack", "dense text"):
            for lim in (2, 3, 0):
                cta_limit(A, lim)
                assert scan_grid(A, total)[0] == min(lim or _sm_count(), tiles)
                _check_scan(A, batch, want, f"{what}, limit {lim}")
        if what == "dense text":
            assert len(want) > 2 * d.size                                         # several keys end at every letter


def _sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def test_ring_cells_cover_every_instantiation():
    assert {cell_instantiation(c) for c in RING_CELLS} == all_instantiations()
    assert {c.log1 for c in RING_CELLS if c.pair and not c.tagmap} == {13, 16, 19, 20}


# ------------------------------------------------------------------ GPU: the end of work at every ring phase
EOW_CELLS = [Cell(1, 4, 1, 16, True), Cell(1, 4, 1, 20, True), Cell(1, 3, 1), Cell(2, 4, 2), Cell(4, 8, 4)]


def _eow_counts(ring):
    S, D = ring.stages, ring.claim_depth
    return sorted({c for c in (1, S - 1, S, S + 1, 2 * S, 2 * S + 1, D - 1, D, D + 1, 2 * D + 1, D + S) if c >= 1})


def _eow_lasts(L, ring):
    """the last tile's bytes: one letter; around 16 (bulk copy against hand copy and zero fill); a slice +- a letter;
    a tile less a letter, a full tile"""
    return sorted({L, 15 // L * L, 16, -(-17 // L) * L, SLICE - L, SLICE + L, ring.tile - L, ring.tile})


def _eow_text(cell, keys, n):
    """sparse text with keys across every half slice, a key starting in the look-ahead of every full tile (its first
    bytes past the tile), and a key ending on the last letter"""
    L = cell.L
    tl = tile_bytes(cell) // L
    t = np.full(n, SPARSE, dtype=np.uint32)
    plant = [k for k in keys if len(k) >= 2]
    for i, b in enumerate(range(SLICE // 2 // L, n, SLICE // 2 // L)):
        k = plant[i % len(plant)]
        st = b - 1 - i % (len(k) - 1)
        if st + len(k) <= n:
            t[st:st + len(k)] = k
    for j, b in enumerate(range(tl, n, tl)):
        k = plant[(3 * j + 1) % len(plant)]
        st = b + j % 4                                            # 0..3 letters: inside the 16 look-ahead bytes
        if st + len(k) <= n:
            t[st:st + len(k)] = k
    k = plant[len(plant) // 2]
    t[max(0, n - len(k)):] = k[max(0, len(k) - n):]
    return t


@pytest.mark.gpu
@pytest.mark.parametrize("cell", EOW_CELLS, ids=[c.name for c in EOW_CELLS])
def test_end_of_work_at_every_ring_phase(cell, monkeypatch, cta_limit):
    keys = _keys(cell, np.random.Generator(np.random.PCG64(_seed(cell))))
    A = _build(cell, keys, monkeypatch)
    _check_shape(A, cell)
    O = _oracle(cell, keys)
    ring = geometry(cell.pair)
    L, dt = cell.L, DT[cell.L]
    counts = _eow_counts(ring)
    reached = set()
    for count in counts:
        for last in _eow_lasts(L, ring):
            n_bytes = (count - 1) * ring.tile + last
            t = _eow_text(cell, keys, n_bytes // L)
            off = np.array([0, t.size], dtype=np.int64)
            batch = (t.astype(dt).view(np.uint8), off * L)
            want = _rows_of(_want(O, cell, t, off))
            for lim in (1, 2, 3):
                cta_limit(A, lim)
                assert scan_grid(A, n_bytes) == (min(lim, count), count)
                _same(rows(A.find_all_batch(batch, algo="filter")), want, f"{count} tiles, last {last} B, limit {lim}")
                reached.add((lim, count))
                for other in (0, lim % 3 + 1):                      # the counter was re-armed for the next launch
                    cta_limit(A, other)
                    _same(rows(A.find_all_batch(batch, algo="filter")), want,
                          f"{count} tiles, last {last} B, limit {other} after limit {lim}")
    assert reached == {(lim, c) for lim in (1, 2, 3) for c in counts}


# ------------------------------------------------------------------ GPU: the full grid at scale
SCALE_CELLS = ([c for c in CELLS if c.pair] +
               [Cell(1, 3, 1), Cell(1, 4, 1), Cell(2, 2, 2), Cell(2, 4, 2), Cell(4, 4, 4)])      # (width, narrow / wide)


@pytest.mark.gpu
@pytest.mark.parametrize("cell", SCALE_CELLS, ids=[c.name for c in SCALE_CELLS])
def test_full_grid_at_scale(cell, monkeypatch):
    """sm_count * stages * 4 tiles: every CTA goes round its ring about 4 times; plants every 4 KiB (every tile
    boundary of both kernels) at rotating residues, dense windows across every 64th tile boundary"""
    sm = _sm_count()
    rng = np.random.Generator(np.random.PCG64(_seed(cell) + 2))
    keys = _keys(cell, rng)
    A = _build(cell, keys, monkeypatch)
    _check_shape(A, cell)
    O = _oracle(cell, keys)
    ring = geometry(cell.pair)
    L, dt = cell.L, DT[cell.L]
    n_tiles = sm * ring.stages * 4
    n = (n_tiles * ring.tile + L * 777) // L
    t = np.full(n, SPARSE, dtype=np.uint32)
    plant = [k for k in keys if len(k) >= 2]
    for i, b in enumerate(range(4096 // L, n, 4096 // L)):
        k = plant[i % len(plant)]
        st = b - 1 - i % (len(k) - 1)
        t[st:st + len(k)] = k
    tl, sl = ring.tile // L, SLICE // L
    for b in range(64 * tl, n - 2 * sl, 64 * tl):
        t[b - 3 * sl // 2:b + 3 * sl // 2] = _alternate(cell, 3 * sl)
    off = np.array([0, n], dtype=np.int64)
    batch = (t.astype(dt).view(np.uint8), off * L)
    assert scan_grid(A, n * L) == (sm, n_tiles + 1)
    want = _rows_of(_want(O, cell, t, off))
    got = rows(A.find_all_batch(batch, algo="filter"))
    assert len(want) > n * L // 4096
    _same(got, want, "filter")
    _same(rows(A.find_all_batch(batch, algo="dfa")), got, "dfa against filter")


# ------------------------------------------------------------------ GPU: grid-stride loops at one SM
TURNS = 4 * 16 * 256              # four turns of every block of a loop bounded by 16 blocks of 256 threads per SM
OUT_TILES = 4 * 8                 # four turns of every block of the replace write pass / stream gather (8 blocks per SM)


def _is_word(case):
    if CASES[case][0] == "bytes":
        return lambda v: re.fullmatch(rb"\w", bytes([v])) is not None
    return lambda v: re.fullmatch(r"\w", chr(v)) is not None


def _letters(case, item):
    if CASES[case][1]:
        return list(item)
    return list(item) if isinstance(item, bytes) else [ord(c) for c in item]


def _grid_case(case, rng, n_letters):
    """keys of one to four letters over the case's alphabet and space (a one-letter key: records at a quarter of the
    letters), and about n_letters of text in 40 haystacks"""
    al = CASES[case][2] + [0x20]
    keys = [[al[0]]] + sorted({tuple(int(x) for x in rng.choice(al, size=int(rng.integers(2, 5)))) for _ in range(10)})
    keys = [list(k) for k in dict.fromkeys(map(tuple, keys))]
    hays = [[int(x) for x in rng.choice(al, size=int(rng.integers(n_letters // 60, n_letters // 26)))] for _ in range(40)]
    return keys, hays


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES))
def test_grid_stride_loops_at_one_sm(case, cta_limit):
    rng = np.random.default_rng(sum(case.encode()) * 31)
    fl, seq, _ = CASES[case]
    width = 4 if fl == "unicode" else (2 if seq else 1)              # bytes per letter of the widest batch
    keys, hays = _grid_case(case, rng, (OUT_TILES * 4096 * 5 // 4) // min(width, 2))
    A, O = automaton(fl, seq, keys)
    cta_limit(A, 1)
    kl = [len(k) for k in keys]
    objs = [obj(fl, seq, h) for h in hays]
    full = oracle_full(O, hays, case)
    chosen = emul_leftmost.greedy(full, kl)
    assert len(full) >= TURNS and len(chosen) >= TURNS
    assert np.array_equal(rows(A.find_all_batch(objs)), _rows_of(full))
    assert np.array_equal(rows(A.find_leftmost_longest_batch(objs)), _rows_of(chosen))
    reps = [list(k) * 2 if i % 3 else [] for i, k in enumerate(keys)]
    R = A.replacer({obj(fl, seq, k): obj(fl, seq, r) for k, r in zip(keys, reps)})
    by_hay = [[(e, k) for h2, e, k in chosen if h2 == h] for h in range(len(hays))]
    want_rep = [emul_replace.definition(hay, c, kl, reps) for hay, c in zip(hays, by_hay)]
    assert sum(map(len, want_rep)) * min(width, 2) >= OUT_TILES * 4096
    assert [_letters(case, x) for x in R.replace_batch(objs)] == want_rep
    if not seq:
        kept = emul_words.definition(hays, full, kl, _is_word(case))
        kept_ll = emul_leftmost.greedy(kept, kl)                     # the word flags run over all len(full) records
        assert np.array_equal(rows(A.find_all_batch(objs, whole_words=True)), _rows_of(kept))
        assert np.array_equal(rows(A.find_leftmost_longest_batch(objs, whole_words=True)), _rows_of(kept_ll))
        by_hay = [[(e, k) for h2, e, k in kept_ll if h2 == h] for h in range(len(hays))]
        assert [_letters(case, x) for x in R.replace_batch(objs, whole_words=True)] == \
            [emul_replace.definition(hay, c, kl, reps) for hay, c in zip(hays, by_hay)]
        ws = [(h, e, v) for h, o in enumerate(objs) for e, v in O.iter(o, ignore_white_space=True)]
        assert len(ws) >= TURNS
        assert np.array_equal(rows(A.find_all_batch(objs, ignore_white_space=True)), _rows_of(ws))
    _stream_chains(case, A, R, keys, reps, rng, width)


def _stream_chains(case, A, R, keys, reps, rng, width):
    """find_all, leftmost, replacing and (for text) word streams: 16 streams fed in three rounds, each feed staging at
    least OUT_TILES gather tiles, against the definitions over each stream's whole text"""
    fl, seq, al = CASES[case]
    al = al + [0x20]
    sw = 4 if fl == "unicode" else (2 if seq else 1)                 # streams of the unicode flavour: 4 bytes per letter
    per = OUT_TILES * 4096 * 5 // 4 // sw // 16
    texts = [[[int(x) for x in rng.choice(al, size=per + int(rng.integers(0, 64)))] for _ in range(3)] for _ in range(16)]
    whole = [sum(parts, []) for parts in texts]
    kl = [len(k) for k in keys]
    _, O = automaton(fl, seq, keys)
    full = [[(e, k) for _, e, k in oracle_full(O, [w], case)] for w in whole]
    ll = [emul_leftmost.greedy([(0, e, k) for e, k in f], kl) for f in full]
    kinds = [("find_all", A.stream_batch(16), full), ("leftmost", A.stream_batch(16, leftmost_longest=True),
                                                      [[(e, k) for _, e, k in x] for x in ll])]
    if not seq:
        isw = _is_word(case)
        kept = [[(e, k) for _, e, k in emul_words.definition([w], [(0, e, k) for e, k in f], kl, isw)] for w, f in zip(whole, full)]
        kinds.append(("words", A.stream_batch(16, whole_words=True), kept))
    for name, B, want in kinds:
        got = [[] for _ in whole]
        for r in range(3):
            m = B.feed([obj(fl, seq, parts[r]) for parts in texts])
            for s, e, k in zip(m.hay_id.tolist(), m.end_index.tolist(), m.key_id.tolist()):
                got[s].append((e, k))
        if name != "find_all":
            m = B.finish(list(range(16)))
            for s, e, k in zip(m.hay_id.tolist(), m.end_index.tolist(), m.key_id.tolist()):
                got[s].append((e, k))
        assert got == want, name
    S = R.stream_batch(16)
    out = [[] for _ in whole]
    for r in range(3):
        for s, x in enumerate(S.feed([obj(fl, seq, parts[r]) for parts in texts])):
            out[s] += _letters(case, x)
    for s, x in enumerate(S.finish(list(range(16)))):
        out[s] += _letters(case, x)
    assert out == [emul_replace.definition(w, [(e, k) for _, e, k in c], kl, reps) for w, c in zip(whole, ll)]
