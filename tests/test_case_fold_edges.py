"""ascii_case_insensitive=True at the edges where a fold goes wrong: every letter of the fold kernel's blocks and tail,
every filter shape on a folded table, the grid-stride loops of the fold, the alias expansion and the batch features at
one SM, the pipelined host route at its 32 MiB chunk and scan cuts, the alias expansion's record bounds, sort keys of 64
and 65 bits with case variants, and batches past 2^31 bytes.

The reference is the same everywhere: the text and the keys folded in numpy (emul_fold.fold), one representative per
group of keys that fold to one text (emul_fold.groups), the C oracle over the folded text; then the aliases added after
their representative (emul_fold.alias_csr / expand), the leftmost selections and the replacement of emul_fold's
definitions, and the word test on the text as given (emul_fold.whole_words).  At 100 MiB and past 2 GiB the records
are also known by construction (the planted keys in a text of no key letter).

  CPU   the vectorised reference against emul_fold's definitions, the numpy fold against the definition, the folded
        cell tables' forced shapes and their coverage of every scan instantiation, the cells' plants at their tiles.
  GPU   (-m gpu) the real routes against the reference.
"""
import ctypes

import numpy as np
import pytest

import emul_fold as ef
import oracle
import pyahocorasick_b200 as pkg
from pyahocorasick_b200 import _native as N
from batch_cases import CASES, DT, check_host_capacities, obj, rows
from kernel_cells import (CELLS, SLICE, _diff, _keys, _ragged, _seed, _text, all_instantiations, cell_instantiation,
                          instantiation, tile_bytes)
from kernel_cells import _check_shape as _check_cell_shape

MiB = 1 << 20
CHUNK = 32 * MiB                  # scan_host_pipelined's chunk; host batches of 48 MiB and more take that path
GUARD = 64
TURNS = 4 * 16 * 256              # four turns of every block of a loop bounded by 16 blocks of 256 threads per SM
OUT_TILES = 4 * 8                 # four turns of every block of the replace write pass / stream gather (8 blocks per SM)
FOLD_CELLS = [c for c in CELLS if c.L in (1, 4)]          # acb_table_upload_folded refuses 2-byte letters
U141 = 0x141                      # Ł: 0x41 in its low byte, never folded


# ------------------------------------------------------------------ the reference
def fold(a):
    """emul_fold.fold keeping the array's dtype (uint8 or uint32 letters), for texts of hundreds of MiB"""
    a = np.asarray(a)
    return np.where((a >= 0x41) & (a <= 0x5A), a + a.dtype.type(0x20), a)


def swap(k):
    """a key with the case of its ASCII letters swapped"""
    return tuple(x ^ 0x20 if 0x41 <= (x & ~0x20) <= 0x5A else x for x in k)


def mixcase(a, rng, p=0.5):
    """the letters with each ASCII letter's case flipped with probability p"""
    a = np.array(a, copy=True)
    low = a | 0x20
    flip = (low >= 0x61) & (low <= 0x7A) & (a < 0x80) & (rng.random(a.shape) < p)
    a[flip] ^= 0x20
    return a


def pick(full, kl, first):
    """leftmost-first (first) or leftmost-longest over (n, 3) representative records: per haystack, p = 0; of the matches
    starting at or after p, the leftmost, then the lowest key id (first) or the longest; p = its end + 1"""
    full = np.asarray(full, dtype=np.int64).reshape(-1, 3)
    if len(full) == 0:
        return full
    hay, end, key = full[:, 0], full[:, 1], full[:, 2]
    ln = kl[key]
    start = end - ln + 1
    o = np.lexsort((key if first else -ln, start, hay))
    hay, start, ln, end, key = hay[o], start[o], ln[o], end[o], key[o]
    head = np.ones(len(o), dtype=bool)
    head[1:] = (hay[1:] != hay[:-1]) | (start[1:] != start[:-1])
    hay, start, ln, end, key = hay[head], start[head], ln[head], end[head], key[head]
    at = hay * (np.int64(1) << 32) + start
    nxt = np.searchsorted(at, at + ln)
    ok = nxt < len(at)
    ok[ok] = hay[nxt[ok]] == hay[ok]
    nx = np.where(ok, nxt, -1).tolist()
    chosen = []
    for i in np.nonzero(np.r_[True, hay[1:] != hay[:-1]])[0].tolist():
        while i >= 0:
            chosen.append(i)
            i = nx[i]
    c = np.array(sorted(chosen), dtype=np.int64)
    return np.stack([hay[c], end[c], key[c]], axis=1)


class Ref:
    """The reference of one key set (letters per key id): with fold, the C oracle over the folded representatives and the
    alias lists; without, the C oracle over the keys as given.  L: 1 for bytes-flavour text (bytes keys, scan_batch_bytes),
    4 for code points (tuple keys, scan_batch_letters)."""

    def __init__(self, keys, L, fold_keys=True):
        self.keys = [tuple(int(x) for x in k) for k in keys]
        self.L = L
        self.kl = np.array(ef.key_lengths(self.keys), dtype=np.int64)
        if fold_keys:
            self.rep, _ = ef.groups(self.keys)
            self.ptr, self.ids = ef.alias_csr(self.keys)
        else:
            self.rep = {i: i for i in range(len(self.keys))}
            self.ptr, self.ids = np.zeros(len(self.keys) + 1, dtype=np.int64), np.empty(0, dtype=np.int64)
        self.fold = fold_keys
        self.O = oracle.OracleAutomaton()
        for kid, k in enumerate(self.keys):
            if self.rep[kid] == kid:
                f = ef.fold(k).tolist() if fold_keys else list(k)
                self.O.add_word(bytes(f) if L == 1 else tuple(f), kid)
        self.O.make_automaton()

    def reps(self, letters, off):
        """(n, 3) int64: the representatives' matches over the (folded) letters cut at off (in letters), reference order"""
        t = fold(letters) if self.fold else np.asarray(letters)
        if self.L == 1:
            r = self.O.scan_batch_bytes(t.astype(np.uint8), np.asarray(off, dtype=np.int64))
        else:
            r = self.O.scan_batch_letters(t.astype(np.uint32), np.asarray(off, dtype=np.int64))
        return np.asarray(r, dtype=np.int64).reshape(-1, 3)

    def expand(self, r):
        """every record followed by the aliases of its key, ascending (emul_fold.expand, vectorised)"""
        r = np.asarray(r, dtype=np.int64).reshape(-1, 3)
        if not len(self.ids) or not len(r):
            return r
        k = r[:, 2]
        inside = k < len(self.ptr) - 1
        cnt = np.ones(len(r), dtype=np.int64)
        cnt[inside] += self.ptr[k[inside] + 1] - self.ptr[k[inside]]
        out = np.repeat(r, cnt, axis=0)
        j = np.arange(len(out)) - np.repeat(np.cumsum(cnt) - cnt, cnt) - 1
        a = j >= 0
        out[a, 2] = self.ids[self.ptr[out[a, 2]] + j[a]]
        return out

    def find_all(self, letters, off):
        return self.expand(self.reps(letters, off))

    def leftmost(self, letters, off, first, is_word=None, hays=None):
        full = self.reps(letters, off)
        if is_word is not None:
            full = self.words(hays, full, is_word)
        return pick(full, self.kl, first)

    def words(self, hays, full, is_word):
        kept = ef.whole_words(hays, [tuple(x) for x in np.asarray(full).tolist()], self.kl, is_word)
        return np.asarray(kept, dtype=np.int64).reshape(-1, 3)

    def replace(self, hays, chosen, reps):
        by = [[] for _ in hays]
        for h, e, k in np.asarray(chosen).tolist():
            by[h].append((e, k))
        return [ef.replaced(list(hay), c, self.kl, reps) for hay, c in zip(hays, by)]


def _same(got, want, what):
    got, want = np.asarray(got, dtype=np.int64).reshape(-1, 3), np.asarray(want, dtype=np.int64).reshape(-1, 3)
    if not np.array_equal(got, want):
        pytest.fail(f"{what}: {_diff([tuple(x) for x in got.tolist()], [tuple(x) for x in want.tolist()])}")


def _same_set(got, want, what):
    _same(np.unique(np.asarray(got, dtype=np.int64).reshape(-1, 3), axis=0),
          np.unique(np.asarray(want, dtype=np.int64).reshape(-1, 3), axis=0), what)
    assert len(got) == len(want), what


def letters_of(fl, x):
    return list(x) if isinstance(x, (bytes, bytearray)) else [ord(c) for c in x]


def build(fl, keys, mp=None, env=None, tagmap=False):
    """the Automaton (STORE_INTS, value = key id) over keys given as letters; env forces ACB_FILTER (and tagmap
    ACB_FORCE_TAGMAP) around make_automaton and the build of the folded host tries"""
    mod = pkg.flavour(fl)
    A = mod.Automaton(mod.STORE_INTS)
    for i, k in enumerate(keys):
        A.add_word(obj(fl, False, k), i)
    if env is None:
        A.make_automaton()
        return A
    with mp.context() as m:
        m.setenv("ACB_FILTER", env)
        if tagmap:
            m.setenv("ACB_FORCE_TAGMAP", "1")
        else:
            m.delenv("ACB_FORCE_TAGMAP", raising=False)
        A.make_automaton()
        A._fold_host(False)
        if A._UNICODE:
            A._fold_host(True)
    return A


def fold_shape(A, narrow=False):
    """filter_shape() of the folded host trie"""
    fv = N.FlatView()
    N.check(A._lib.acb_trie_flat_view(A._fold_host(narrow).trie, ctypes.byref(fv)))
    return dict(gram_bytes=fv.gram_bytes, stride=fv.stride, log2_bits1=fv.log2_bits1, log2_bits2=fv.log2_bits2,
                log2_bits3=fv.log2_bits3, log2_anchor_slots=fv.log2_anchor_slots, filter_flags=fv.filter_flags)


class _Shape:
    def __init__(self, fs):
        self.fs = fs

    def filter_shape(self):
        return self.fs


@pytest.fixture
def cta_limit():
    """limit(A, n): the CTA limit of every device-0 table of A -- the full and latin-1 ones and the folded ones of both
    widths; every table is set back to 0 after (A is kept alive until then: its tables go with it)"""
    seen = []

    def limit(A, n):
        tbs = [A._ensure_table(0)]
        if A._UNICODE:
            core = A._ensure_narrow(0)
            if core is not None:
                tbs.append(core[1])
        for narrow in (False, True) if A._UNICODE else (False,):
            tb = A._table_for(0, narrow, True)
            if tb is not None:
                tbs.append(tb)
        for tb in tbs:
            N.check(N.lib().acb_table_set_cta_limit(tb, n))
            seen.append((A, tb))
    yield limit
    for _, tb in seen:
        N.check(N.lib().acb_table_set_cta_limit(tb, 0))


def scan_grid(tb, total_bytes):
    grid, tiles = ctypes.c_int32(), ctypes.c_int64()
    N.check(N.lib().acb_table_scan_grid(tb, int(total_bytes), ctypes.byref(grid), ctypes.byref(tiles)))
    return grid.value, tiles.value


def launches(call):
    L = N.lib()
    before = L.acb_launch_count()
    out = call()
    return L.acb_launch_count() - before, out


# ------------------------------------------------------------------ CPU: the reference
def _small_case(rng, al, n_keys, n_hays):
    keys = []
    for _ in range(n_keys):
        k = tuple(int(x) for x in rng.choice(al, size=int(rng.integers(1, 5))))
        for v in ([k, swap(k)] if rng.integers(0, 2) else [k]):
            if v not in keys:
                keys.append(v)
    hays = [[int(x) for x in rng.choice(al, size=int(rng.integers(0, 40)))] for _ in range(n_hays)]
    return keys, hays


@pytest.mark.parametrize("L", [1, 4])
def test_reference_is_emul_folds_definitions(L):
    """the vectorised reference (oracle over folded representatives, numpy expansion, leftmost walk) against emul_fold"""
    rng = np.random.default_rng(40 + L)
    al = [0x61, 0x41, 0x62, 0x42, 0x40, 0x5B, 0x60, 0x7B] + ([0xC1, 0xE1] if L == 1 else [U141, 0x161, 0x1F641])
    for _ in range(120):
        keys, hays = _small_case(rng, al, int(rng.integers(1, 8)), int(rng.integers(1, 5)))
        R = Ref(keys, L)
        letters = np.array([x for h in hays for x in h], dtype=np.uint32)
        off = np.concatenate([[0], np.cumsum([len(h) for h in hays])]).astype(np.int64)
        assert [tuple(x) for x in R.find_all(letters, off).tolist()] == ef.find_all(keys, hays), (keys, hays)
        is_word = {0x61, 0x42}.__contains__
        for first in (True, False):
            assert [tuple(x) for x in R.leftmost(letters, off, first).tolist()] == ef.leftmost(keys, hays, first)
            assert [tuple(x) for x in R.leftmost(letters, off, first, is_word, hays).tolist()] == \
                ef.leftmost(keys, hays, first, is_word)
            reps = [[0x5F] * (i % 3) for i in range(len(keys))]
            assert R.replace(hays, R.leftmost(letters, off, first), reps) == ef.replace(keys, reps, hays, first)
        got, total = ef.expand(R.reps(letters, off), R.ptr, R.ids, 10 ** 6)
        assert np.array_equal(got, R.expand(R.reps(letters, off))) and total == len(got)


def test_fold_keeps_dtype_and_is_the_definition():
    b = np.arange(256, dtype=np.uint8)
    assert fold(b).dtype == np.uint8 and np.array_equal(fold(b), ef.fold(b))
    w = np.array([0x40, 0x41, 0x5A, 0x5B, 0x60, 0x7B, U141, 0x15A, 0x1F641, 0x10FFFF], dtype=np.uint32)
    assert fold(w).dtype == np.uint32 and np.array_equal(fold(w), ef.fold(w))
    assert swap((0x61, 0x5A, 0x40, 0x7B, U141, 0xE1)) == (0x41, 0x7A, 0x40, 0x7B, U141, 0xE1)


# ------------------------------------------------------------------ the folded cells
def cell_keys(cell, rng):
    """kernel_cells' keys of the cell, then the swapcase() variant of every third key that has an ASCII letter (groups,
    so the find_all routes expand), and for 4-byte letters a key starting with U+0141"""
    keys = _keys(cell, rng)
    variants = [swap(k) for k in keys[::3] if swap(k) != k]
    keys = keys + [v for v in dict.fromkeys(variants) if v not in keys]
    if cell.L == 4:
        keys.append((U141,) + keys[0][1:])
    return keys


def cell_text(cell, keys, rng, n_bytes):
    """_text's plants across every lane run, slice and tile boundary, every ASCII letter in random case; 4-byte letters:
    U+0141 before every third boundary plant and the U+0141 key planted after every tenth"""
    t, starts = _text(cell, keys, rng, n_bytes)
    t = mixcase(t, rng)
    if cell.L == 4:
        u = keys[-1]
        for i, st in enumerate(starts.tolist()):
            if i % 3 == 0 and st > 0:
                t[st - 1] = U141
            if i % 10 == 5 and st + 40 + len(u) < t.size:
                t[st + 40:st + 40 + len(u)] = u
    return t, starts


def cell_automaton(cell, keys, mp):
    fl = "unicode" if cell.L == 4 else "bytes"
    A = build(fl, keys, mp, cell.env, cell.tagmap)
    fs = fold_shape(A)
    _check_cell_shape(_Shape(fs), cell)
    return A, fs


def test_folded_cells_reach_every_instantiation(monkeypatch):
    """the folded tables of the 1- and 4-byte cells, forced while the folded trie is built, select all 40 stream and 2
    pair instantiations and the pair kernel with the tag bitmap"""
    seen = set()
    for cell in FOLD_CELLS:
        keys = cell_keys(cell, np.random.Generator(np.random.PCG64(_seed(cell))))
        A, fs = cell_automaton(cell, keys, monkeypatch)
        assert len(A._fold_host(False).alias_ids) > 0                    # every cell has case variants
        seen.add(instantiation(fs))
        if cell.pair and fs["log2_bits3"]:
            seen.add(("pair-tagmap",))
        assert cell_instantiation(cell) in seen
    assert seen == all_instantiations(), sorted(all_instantiations() ^ seen, key=str)


@pytest.mark.parametrize("cell", FOLD_CELLS, ids=[c.name for c in FOLD_CELLS])
def test_cell_plants_and_reference(cell):
    """the cell's mixed-case text plants at its kernel's tile (the last three boundary plants start just before 1, 2
    and 3 tiles), and on 2 KiB of it the reference equals emul_fold's definitions"""
    rng = np.random.Generator(np.random.PCG64(_seed(cell)))
    keys = cell_keys(cell, rng)
    tile = tile_bytes(cell)
    _, starts = cell_text(cell, keys, rng, 3 * tile + 4 * SLICE)
    at = starts[-3:] * cell.L
    assert all(j * tile - 256 < a < j * tile for j, a in zip((1, 2, 3), at)), (tile, at.tolist())
    t, _ = cell_text(cell, keys, rng, 2048 + cell.L * 53)
    cut = t.size // 3
    hays = [t[:cut].tolist(), t[cut:].tolist()]
    off = np.array([0, cut, t.size], dtype=np.int64)
    R = Ref(keys, cell.L)
    want = ef.find_all(keys, hays)
    assert [tuple(x) for x in R.find_all(t, off).tolist()] == want
    assert len(R.ids) and any(k in set(R.ids.tolist()) for _, _, k in want)      # aliases occur in the text
    if cell.L == 4:
        assert any(k == len(keys) - 1 for _, _, k in want)                      # the U+0141 key is found unfolded
    for first in (True, False):
        assert [tuple(x) for x in R.leftmost(t, off, first).tolist()] == ef.leftmost(keys, hays, first)


# ------------------------------------------------------------------ GPU: 1. the fold, letter by letter
BYTE_KEYS = [(b,) for b in range(256) if not 0x41 <= b <= 0x5A]
WIDE_TRAPS = [U141, 0x161, 0xC1, 0x1F641, 0x40, 0x5B, 0x60, 0x7B]
WIDE_KEYS = [(x,) for x in range(0x61, 0x7B)] + [(x,) for x in WIDE_TRAPS] + [(0x100,), (0x1F600,)]


def _per_letter_want(ids, folded, off):
    """a record at every letter that folds to a key: (haystack, end, the key id of its folded letter)"""
    off = np.asarray(off, dtype=np.int64)
    pos = np.nonzero((ids >= 0)[folded])[0]
    hay = np.searchsorted(off, pos, side="right") - 1
    return np.stack([hay, pos - off[hay], ids[folded[pos]]], axis=1)


@pytest.mark.gpu
@pytest.mark.parametrize("L", [1, 4])
def test_gpu_fold_letter_by_letter(L, cta_limit):
    """Every byte value but A-Z (1-byte letters), or a-z and traps (4-byte letters), as one-letter keys: no aliases, and
    find_all reports at every letter the key of its folded letter.  Batches of every total that gives n16 = 0..5 blocks
    and each tail residue, as a host list and a CUDA tensor (left unchanged); then four turns of every fold block at
    limit 1 and at the full grid, with a ragged tail."""
    import torch
    fl = "bytes" if L == 1 else "unicode"
    keys = BYTE_KEYS if L == 1 else WIDE_KEYS
    A = build(fl, keys)
    assert not len(A._fold_host(False).alias_ids)
    ids = np.full(0x110000 if L == 4 else 256, -1, dtype=np.int64)
    for i, (x,) in enumerate(keys):
        ids[x] = i
    rng = np.random.default_rng(L)
    pool = np.arange(256) if L == 1 else np.array([x for (x,) in keys] + [x - 0x20 for x in range(0x61, 0x7B)])
    for n in range(1, 81):
        if L == 4 and n % 4:
            continue
        letters = rng.choice(pool, size=n // L if L == 4 else n)
        if L == 4:
            letters[:len(WIDE_TRAPS)] = WIDE_TRAPS[:len(letters)]
        cut = len(letters) // 3
        off = np.array([0, cut, len(letters)], dtype=np.int64)
        want = _per_letter_want(ids, fold(letters), off)
        assert len(want) == len(letters)
        objs = [obj(fl, False, letters[:cut].tolist()), obj(fl, False, letters[cut:].tolist())]
        _same(rows(A.find_all_batch(objs, ascii_case_insensitive=True)), want, f"{n} bytes, list")
        raw = letters.astype(DT[L]).view(np.uint8)
        d = torch.from_numpy(raw.reshape(1, -1).copy()).cuda()
        _same(rows(A.find_all_batch(d, ascii_case_insensitive=True)), _per_letter_want(ids, fold(letters), [0, len(letters)]),
              f"{n} bytes, tensor")
        assert np.array_equal(d.cpu().numpy().reshape(-1), raw)
    # four turns of the four-block loop: 16 blocks of 256 threads at limit 1, 16 per SM at the full grid
    for lim in (1, 0):
        sm = 1 if lim else torch.cuda.get_device_properties(0).multi_processor_count
        blocks16 = 4 * 4 * 16 * 256 * sm + 3                      # 16-byte blocks, and a few more for the short loop
        n = (blocks16 * 16 + 12) // L                             # a tail of 12 bytes
        letters = rng.choice(pool.astype(DT[L]), size=n)
        if lim == 0:                                              # sparse: a record at about one letter in 40
            cold = rng.integers(0, 40, size=n, dtype=np.uint8) != 0
            letters[cold] = 0x30 + rng.integers(0, 3, size=int(cold.sum()), dtype=np.uint8)
        letters[-3:] = [0x5A, 0x41, 0x5A]                         # capitals in the tail
        if lim == 0:
            keep = np.array([i for i, (x,) in enumerate(keys) if x not in (0x30, 0x31, 0x32)])
            sub = [keys[i] for i in keep]
            A = build(fl, sub)
            ids = np.full(ids.size, -1, dtype=np.int64)
            for i, (x,) in enumerate(sub):
                ids[x] = i
        cta_limit(A, lim)
        raw = letters.astype(DT[L]).view(np.uint8)
        off = np.array([0, n // 2, n], dtype=np.int64)
        f = fold(letters)
        _same(rows(A.find_all_batch((raw, off * L), ascii_case_insensitive=True)), _per_letter_want(ids, f, off),
              f"limit {lim}, host")
        d = torch.from_numpy(raw.reshape(1, -1).copy()).cuda()
        _same(rows(A.find_all_batch(d, ascii_case_insensitive=True)), _per_letter_want(ids, f, [0, n]), f"limit {lim}, tensor")
        assert torch.equal(d.reshape(-1).cpu(), torch.from_numpy(raw))
        del d


# ------------------------------------------------------------------ GPU: 2. every filter shape on a folded table
_RAN = set()


def _check_methods(A, R, batch, letters, off, what, algos=("filter", "dfa"), replace=None):
    want = R.find_all(letters, off)
    for algo in algos:
        _same(rows(A.find_all_batch(batch, algo=algo, ascii_case_insensitive=True)), want, f"{what}, find_all {algo}")
    _same_set(rows(A.find_all_batch(batch, algo="filter", sort=False, ascii_case_insensitive=True)), want,
              f"{what}, find_all unsorted")
    for first in (True, False):
        m = A.find_leftmost_first_batch if first else A.find_leftmost_longest_batch
        _same(rows(m(batch, algo=algos[0], ascii_case_insensitive=True)), R.leftmost(letters, off, first),
              f"{what}, leftmost-{'first' if first else 'longest'}")
    return want


@pytest.mark.gpu
@pytest.mark.parametrize("cell", FOLD_CELLS, ids=[c.name for c in FOLD_CELLS])
def test_gpu_folded_cell(cell, monkeypatch):
    """mixed-case keys of the cell planted in mixed case across every boundary of its kernel, with case variants of a
    third of the keys: one haystack, a ragged batch and a fixed stride, filter and DFA, find_all, both selections and
    replacement of both kinds"""
    rng = np.random.Generator(np.random.PCG64(_seed(cell) + 7))
    keys = cell_keys(cell, rng)
    A, fs = cell_automaton(cell, keys, monkeypatch)
    R = Ref(keys, cell.L)
    L, dt, tile = cell.L, DT[cell.L], tile_bytes(cell)
    t, starts = cell_text(cell, keys, rng, 3 * tile + L * 1291)
    n = t.size
    flat = t.astype(dt).view(np.uint8)
    one = np.array([0, n], dtype=np.int64)
    want = _check_methods(A, R, (flat, one * L), t, one, "one haystack")
    assert len(want) > len(starts) // 2 and len(np.intersect1d(want[:, 2], R.ids))
    fl = "unicode" if L == 4 else "bytes"
    reps = [[0x5F] * (i % 3) + list(k[:1]) for i, k in enumerate(keys)]
    for first in (True, False):
        Rp = A.replacer({obj(fl, False, k): obj(fl, False, r) for k, r in zip(keys, reps)}, leftmost_first=first)
        got, goff = Rp.replace_batch((flat, one * L), ascii_case_insensitive=True)
        assert [np.asarray(got).view(dt).tolist()] == R.replace([t.tolist()], R.leftmost(t, one, first), reps), first
    roff = _ragged(rng, n, starts, np.arange(tile // L, n, tile // L))
    _check_methods(A, R, (flat, roff * L), t, roff, "ragged batch", algos=("filter",))
    _same(rows(A.find_all_batch((flat, roff * L), algo="dfa", ascii_case_insensitive=True)), R.find_all(t, roff), "ragged, dfa")
    k = flat.size // 512
    soff = np.arange(k + 1, dtype=np.int64) * (512 // L)
    _same(rows(A.find_all_batch(flat[:k * 512].reshape(k, 512), ascii_case_insensitive=True)),
          R.find_all(t[:k * (512 // L)], soff), "stride 512")
    _RAN.add(instantiation(fs))
    if cell.pair and fs["log2_bits3"]:
        _RAN.add(("pair-tagmap",))


@pytest.mark.gpu
def test_gpu_every_instantiation_ran_folded(request):
    """the folded cells above, as they ran on the GPU, reached every 1- and 4-byte scan instantiation and the pair kernel
    with and without the tag bitmap (run after them, in one session)"""
    names = {it.name for it in request.session.items}
    if not all(f"test_gpu_folded_cell[{c.name}]" in names for c in FOLD_CELLS):
        pytest.skip("only part of the folded cells was selected")
    assert _RAN == all_instantiations(), sorted(all_instantiations() - _RAN, key=str)


# ------------------------------------------------------------------ GPU: 3. grid-stride loops at one SM
GRID_CASES = {"bytes": ([0x61, 0x41, 0x62, 0x42, 0xE9, 0xC9, 0x20], 1),
              "latin1": ([0x61, 0x41, 0x62, 0x42, 0xE9, 0xC9, 0x20], 4),
              "wide": ([0x61, 0x41, 0x142, U141, 0x1F600, 0x20], 4)}
WORD_LETTERS = [0x61, 0x41, 0x62]


def _grid_keys(al, rng):
    """a one-letter key (records at a third of the letters), two- to four-letter keys, and every case variant of the
    first three (groups of up to 16)"""
    keys = [(0x61,)] + sorted({tuple(int(x) for x in rng.choice(al, size=int(rng.integers(2, 5)))) for _ in range(10)})
    keys = list(dict.fromkeys(keys))
    for k in keys[1:4]:
        for m in range(1, 1 << len(k)):
            v = tuple(x ^ 0x20 if (m >> i) & 1 and 0x41 <= (x & ~0x20) <= 0x5A and x < 0x80 else x for i, x in enumerate(k))
            if v not in keys:
                keys.append(v)
    return keys


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(GRID_CASES))
def test_gpu_grid_stride_loops_at_one_sm(case, cta_limit):
    """At CTA limit 1, with records enough for four turns of every block: the folded find_all with aliases (the
    expansion's count and scatter), both selections, replacement of both kinds, whole words; every folded stream form
    fed in three rounds; and the plain leftmost-first whole-batch, replacer and stream forms."""
    al, L = GRID_CASES[case]
    fl = CASES[case][0]
    rng = np.random.default_rng(sum(case.encode()) * 37)
    keys = _grid_keys(al, rng)
    n_letters = OUT_TILES * 4096 * 5 // 4 // (2 if L == 4 else 1)
    hays = [[int(x) for x in rng.choice(al, size=int(rng.integers(n_letters // 60, n_letters // 26)))] for _ in range(40)]
    A = build(fl, keys)
    assert len(A._fold_host(case == "latin1").alias_ids) >= 3
    cta_limit(A, 1)
    R = Ref(keys, 1 if fl == "bytes" else 4)
    letters = np.array([x for h in hays for x in h], dtype=np.uint32)
    off = np.concatenate([[0], np.cumsum([len(h) for h in hays])]).astype(np.int64)
    objs = [obj(fl, False, h) for h in hays]
    tb = A._table_for(0, case == "latin1", True)
    assert scan_grid(tb, letters.size)[0] == 1
    full = R.find_all(letters, off)
    assert len(full) >= TURNS and len(full) > len(R.reps(letters, off))
    _same(rows(A.find_all_batch(objs, ascii_case_insensitive=True)), full, "find_all")
    reps = [list(k) * 2 if i % 3 else [] for i, k in enumerate(keys)]
    ww = obj(fl, False, WORD_LETTERS)
    is_word = set(WORD_LETTERS).__contains__
    for first in (True, False):
        chosen = R.leftmost(letters, off, first)
        assert len(chosen) >= TURNS
        m = A.find_leftmost_first_batch if first else A.find_leftmost_longest_batch
        _same(rows(m(objs, ascii_case_insensitive=True)), chosen, f"leftmost first={first}")
        Rp = A.replacer({obj(fl, False, k): obj(fl, False, r) for k, r in zip(keys, reps)}, leftmost_first=first)
        want = R.replace(hays, chosen, reps)
        assert sum(map(len, want)) * min(L, 2) >= OUT_TILES * 4096
        assert [letters_of(fl, x) for x in Rp.replace_batch(objs, ascii_case_insensitive=True)] == want, first
        kept = R.leftmost(letters, off, first, is_word, hays)
        _same(rows(m(objs, whole_words=ww, ascii_case_insensitive=True)), kept, f"leftmost words first={first}")
        assert [letters_of(fl, x) for x in Rp.replace_batch(objs, whole_words=ww, ascii_case_insensitive=True)] == \
            R.replace(hays, kept, reps), first
    _same(rows(A.find_all_batch(objs, whole_words=ww, ascii_case_insensitive=True)),
          R.expand(R.words(hays, R.reps(letters, off), is_word)), "find_all words")
    # the plain leftmost-first forms at one SM
    P = Ref(keys, R.L, fold_keys=False)
    chosen = P.leftmost(letters, off, True)
    assert len(chosen) >= TURNS
    _same(rows(A.find_leftmost_first_batch(objs)), chosen, "plain leftmost-first")
    Rf = A.replacer({obj(fl, False, k): obj(fl, False, r) for k, r in zip(keys, reps)}, leftmost_first=True)
    assert [letters_of(fl, x) for x in Rf.replace_batch(objs)] == P.replace(hays, chosen, reps)
    _streams(A, keys, reps, R, P, fl, rng, al, L)


def _streams(A, keys, reps, R, P, fl, rng, al, L):
    """16 streams fed in three rounds, each feed staging at least OUT_TILES gather tiles, against each stream's whole
    text: the folded find_all, find_all + words, leftmost-longest, leftmost-first and replacing streams, and the plain
    leftmost-first and leftmost-first replacing streams"""
    per = OUT_TILES * 4096 * 5 // 4 // L // 16
    texts = [[[int(x) for x in rng.choice(al, size=per + int(rng.integers(0, 64)))] for _ in range(3)] for _ in range(16)]
    whole = [sum(parts, []) for parts in texts]
    wl = np.array([x for w in whole for x in w], dtype=np.uint32)
    wo = np.concatenate([[0], np.cumsum([len(w) for w in whole])]).astype(np.int64)
    ww = obj(fl, False, WORD_LETTERS)
    is_word = set(WORD_LETTERS).__contains__

    def per_stream(r):
        out = [[] for _ in whole]
        for h, e, k in np.asarray(r).tolist():
            out[h].append((e, k))
        return out
    kinds = [("find_all", A.ascii_case_insensitive_stream_batch(16), R.find_all(wl, wo), False),
             ("words", A.ascii_case_insensitive_stream_batch(16, whole_words=ww),
              R.expand(R.words(whole, R.reps(wl, wo), is_word)), True),
             ("longest", A.ascii_case_insensitive_stream_batch(16, leftmost_longest=True), R.leftmost(wl, wo, False), True),
             ("first", A.ascii_case_insensitive_stream_batch(16, leftmost_first=True), R.leftmost(wl, wo, True), True),
             ("plain first", A.stream_batch(16, leftmost_first=True), P.leftmost(wl, wo, True), True)]
    for name, B, want, finish in kinds:
        got = [[] for _ in whole]
        for r in range(3):
            m = B.feed([obj(fl, False, parts[r]) for parts in texts])
            for s, e, k in zip(m.hay_id.tolist(), m.end_index.tolist(), m.key_id.tolist()):
                got[s].append((e, k))
        if finish:
            m = B.finish(list(range(16)))
            for s, e, k in zip(m.hay_id.tolist(), m.end_index.tolist(), m.key_id.tolist()):
                got[s].append((e, k))
        assert got == per_stream(want), name
    for first, fold_keys in ((True, True), (False, True), (True, False)):
        Rp = A.replacer({obj(fl, False, k): obj(fl, False, r) for k, r in zip(keys, reps)}, leftmost_first=first)
        S = Rp.ascii_case_insensitive_stream_batch(16) if fold_keys else Rp.stream_batch(16)
        Q = R if fold_keys else P
        out = [[] for _ in whole]
        for r in range(3):
            for s, x in enumerate(S.feed([obj(fl, False, parts[r]) for parts in texts])):
                out[s] += letters_of(fl, x)
        for s, x in enumerate(S.finish(list(range(16)))):
            out[s] += letters_of(fl, x)
        assert out == Q.replace(whole, Q.leftmost(wl, wo, first), reps), (first, fold_keys)


# ------------------------------------------------------------------ GPU: 4. the pipelined host route on a folded table
PAIR_AT_CUT = ((0x6A, 0x6B, 0x6C, 0x6D, 0x6E, 0x71), (0x71, 0x72, 0x73, 0x74, 0x75, 0x76))    # jklmnq, qrstuv: one q shared
RUN_KEY = (0x7A,) * 7                                                                         # zzzzzzz


def _pipe_keys(rng, L, n=40):
    """PAIR_AT_CUT, RUN_KEY and n mixed-case keys of 5..12 ASCII letters (4-byte letters: some with ł), no two folding to
    one text"""
    al = list(range(0x61, 0x7A)) + ([0x142] if L == 4 else [])           # no z but in RUN_KEY
    keys = [tuple(mixcase(np.array(k), rng).tolist()) for k in PAIR_AT_CUT + (RUN_KEY,)]
    seen = {tuple(ef.fold(k).tolist()) for k in keys}
    while len(keys) < n + 3:
        k = tuple(mixcase(rng.choice(al, size=int(rng.integers(5, 13))), rng).tolist())
        if tuple(ef.fold(k).tolist()) not in seen:
            seen.add(tuple(ef.fold(k).tolist()))
            keys.append(k)
    return keys


def _pipe_batch(rng, keys, L, n, reach, filler):
    """n letters of filler (no key letter) with keys planted in random case every 4093 letters, and at every chunk cut:
    jklmnq ending exactly at the cut and qrstuv starting one letter before it; a run of nine z starting one letter
    before the scan cut (the cut - reach), so that zzzzzzz starts at the scan cut and one letter either side.  4-byte
    letters: U+0141 on both sides of each.  Cut into a ragged batch with one haystack across the chunk cuts 1 and 2 and
    empty haystacks on the other cuts.  Returns the letters, the offsets (in letters), [(start, key id)] of the cut
    plants and the long haystack."""
    t = rng.choice(np.asarray(filler, dtype=np.uint32), size=n)
    cl, rl = CHUNK // L, reach // L
    nch = -(-n * L // CHUNK)
    for i, st in enumerate(range(2048, n - 64, 4093)):
        k = keys[3 + i % (len(keys) - 3)]
        t[st:st + len(k)] = mixcase(np.array(k), rng)
    plants = []
    for c in range(1, nch):
        b, s = c * cl, c * cl - rl
        t[b - 6:b + 5] = mixcase(np.array(PAIR_AT_CUT[0] + PAIR_AT_CUT[1][1:]), rng)
        t[s - 1:s + 8] = mixcase(np.full(9, 0x7A), rng)
        plants += [(b - 6, 0), (b - 1, 1), (s - 1, 2), (s, 2), (s + 1, 2)]
        if L == 4:
            t[[b - 7, b + 5, s - 2, s + 8]] = U141
    k = keys[3]
    t[n - len(k):] = k
    long_hay = (cl // 3, min(2 * cl + cl // 2, n - 1000))
    cuts = [*long_hay] + rng.integers(0, long_hay[0], size=300).tolist() + rng.integers(long_hay[1], n, size=300).tolist()
    for c in range(1, nch):
        if not long_hay[0] < c * cl - rl < long_hay[1]:
            cuts += [c * cl] * 3 + [c * cl - rl] * 2
    off = np.concatenate([[0], np.sort(cuts), [n]]).astype(np.int64)
    return t, off, plants, long_hay


@pytest.mark.gpu
@pytest.mark.parametrize("fl", ["bytes", "unicode"])
def test_gpu_pipelined_host_route(fl):
    """About 100 MiB of 1-byte letters (or 52 MiB of 4-byte ones) in (flat, offsets) form.  Without case variants the
    folded scan takes the pipeline: one fold launch per chunk more than the case-sensitive scan of the same batch.  With
    variants of some keys it takes the one-piece route (fold, scan, expansion, sort).  sort=True and sort=False, against
    the oracle over the folded text, and the cut plants by construction."""
    L = 1 if fl == "bytes" else 4
    rng = np.random.default_rng(444 + L)
    keys = _pipe_keys(rng, L)
    reach = (max(map(len, keys)) * L + 31) & ~31
    n = 100 * MiB + 12345 if L == 1 else (52 * MiB) // 4 + 3
    t, off, plants, long_hay = _pipe_batch(rng, keys, L, n, reach, list(b"0123456789-+") if L == 1 else [0x30, 0x31, 0x1F600, 0xE9])
    assert (n * L) % 16 and n * L >= 48 * MiB
    nch = -(-n * L // CHUNK)
    flat = t.astype(DT[L]).view(np.uint8)
    batch = (flat, off * L)
    for variants in (False, True):
        ks = keys + ([swap(k) for k in keys[::4]] if variants else [])
        A = build(fl, ks)
        R = Ref(ks, L)
        want = R.find_all(t, off)
        have = set(map(tuple, want.tolist()))
        for st, kid in plants:                                           # every cut plant inside a haystack is found
            h = int(np.searchsorted(off, st, side="right")) - 1
            e = st + len(ks[kid]) - 1
            assert (e >= off[h + 1]) or (h, e - off[h], kid) in have, (st, kid)
        assert sum(1 for st, _ in plants if long_hay[0] <= st < long_hay[1] - 16) >= 5 * min(nch - 1, 2)
        h_long = int(np.searchsorted(off, long_hay[0], side="right")) - 1
        ends = want[want[:, 0] == h_long, 1] + long_hay[0]
        assert off[h_long] == long_hay[0]
        assert all(((ends * L >= a) & (ends * L < a + CHUNK)).any() for a in range(0, min(nch, 3) * CHUNK, CHUNK))
        A._match_cap = len(want) + 1024
        A.find_all_batch(batch, ascii_case_insensitive=True)             # every workspace grown
        for sort in (True, False):
            plain, _ = launches(lambda: A.find_all_batch(batch, sort=sort))
            count, m = launches(lambda: A.find_all_batch(batch, sort=sort, ascii_case_insensitive=True))
            if not variants:
                assert count == plain + nch and count == nch * (2 + sort), (count, plain, nch)
            elif not sort:
                assert count == 1 + 1 + 2, count                          # fold, one scan, expansion count + scatter
            if sort:
                _same(rows(m), want, f"variants={variants}")
            else:
                _same_set(rows(m), want, f"variants={variants}, unsorted")


# ------------------------------------------------------------------ GPU: 5. record bounds of the expansion
def _group_keys():
    """64 groups of 1..64 members: group g holds the first g case variants of a six-letter word of its own"""
    keys, reps = [], []
    for g in range(1, 65):
        base = [0x30 + g // 10, 0x30 + g % 10]
        reps.append(len(keys))
        for m in range(g):
            keys.append(tuple(base + [(0x61 + i) ^ (0x20 if (m >> i) & 1 else 0) for i in range(6)]))
    return keys, reps


def _expand(tb, d_in, n, d_out, cap, d_cnt):
    import torch
    return N.lib().acb_expand_aliases_device(tb, d_in.data_ptr() if n else None, n, d_out.data_ptr() if cap else None, cap,
                                             d_cnt.data_ptr(), torch.cuda.current_stream().cuda_stream)


@pytest.mark.gpu
def test_gpu_expansion_never_writes_past_cap(cta_limit):
    """acb_expand_aliases_device over one record of every group, in shuffled order, at every capacity from 0 to
    total + 1 (a cut at every offset inside every group): rows at or past cap keep their fill, *d_count is set to the
    total whatever it held, the input is unchanged; n = 0; four grid-stride turns at limit 1; the refusal of
    n >= 2^31 - 1 before anything is launched"""
    import torch
    keys, reps = _group_keys()
    A = build("bytes", keys)
    R = Ref(keys, 1)
    assert R.ids.size == len(keys) - 64
    A._ensure_table(0)                                                  # its first upload drops the folded tables
    tb = A._table_for(0, False, True)
    rng = np.random.default_rng(65)
    rec = np.array([(int(rng.integers(0, 9)), int(rng.integers(0, 1000)), r) for r in rng.permutation(reps)], dtype=np.int32)
    d_in = torch.from_numpy(rec).cuda()
    want = R.expand(rec)
    total = len(want)
    assert total == 64 * 65 // 2
    for cap in range(total + 2):
        out = torch.full((cap + GUARD, 3), -7, dtype=torch.int32, device="cuda")
        cnt = torch.tensor([(cap * 7919) % 100003 - 5], dtype=torch.int64, device="cuda")
        N.check(_expand(tb, d_in, len(rec), out, cap, cnt))
        o = out.cpu().numpy()
        assert int(cnt.item()) == total, cap
        assert (o[cap:] == -7).all(), cap
        assert np.array_equal(o[:min(cap, total)], want[:cap]), cap
    assert np.array_equal(d_in.cpu().numpy(), rec)
    cnt = torch.tensor([99], dtype=torch.int64, device="cuda")
    out = torch.full((GUARD, 3), -7, dtype=torch.int32, device="cuda")
    N.check(_expand(tb, d_in, 0, out, 0, cnt))
    assert int(cnt.item()) == 0 and (out.cpu().numpy() == -7).all()
    # four grid-stride turns of the count and scatter kernels in one SM
    cta_limit(A, 1)
    big = np.array([(i % 50, i, reps[int(x)]) for i, x in enumerate(rng.integers(0, 64, size=4 * TURNS + 17))], dtype=np.int32)
    d_big = torch.from_numpy(big).cuda()
    want = R.expand(big)
    for cap in (len(want), len(want) // 2 + 1):
        out = torch.full((cap + GUARD, 3), -7, dtype=torch.int32, device="cuda")
        cnt = torch.tensor([-1], dtype=torch.int64, device="cuda")
        N.check(_expand(tb, d_big, len(big), out, cap, cnt))
        o = out.cpu().numpy()
        assert int(cnt.item()) == len(want) and (o[cap:] == -7).all() and np.array_equal(o[:cap], want[:cap])
    # n = 2^31 - 1 and more: refused before anything is allocated or launched (the buffers are never read)
    torch.cuda.synchronize()
    cnt = torch.tensor([42], dtype=torch.int64, device="cuda")
    for n in ((1 << 31) - 1, 1 << 31):
        before = N.lib().acb_launch_count()
        assert _expand(tb, d_big, n, out, 1, cnt) == N.ACB_ERANGE
        assert N.lib().acb_launch_count() == before
    torch.cuda.synchronize()
    assert int(cnt.item()) == 42


@pytest.mark.gpu
def test_gpu_folded_routes_report_exact_overflow():
    """the host find_all route of a folded table with aliases, with and without words: ACB_EOVERFLOW with the exact
    expanded count at capacities 0, 1, n - 1, the records at n; the device route through the Python retry"""
    import torch
    keys, _ = _group_keys()
    keys = keys[:3 + 4] + [tuple(b"ab"), tuple(b"AB"), tuple(b"aB"), tuple(b"b")]
    A = build("bytes", keys)
    R = Ref(keys, 1)
    rng = np.random.default_rng(3)
    hays = [mixcase(np.frombuffer(b"ab 02abcdef 03abc " * 30, dtype=np.uint8), rng).tolist() for _ in range(6)] + [[]]
    letters = np.array([x for h in hays for x in h], dtype=np.uint8)
    off = np.concatenate([[0], np.cumsum([len(h) for h in hays])]).astype(np.int64)
    A._ensure_table(0)                                                  # its first upload drops the folded tables
    tb = A._table_for(0, False, True)
    want = R.find_all(letters, off)
    assert len(want) > 200 and len(want) > len(R.reps(letters, off))
    check_host_capacities(lambda out, cap, found: N.lib().acb_scan_host(tb, N.ptr(letters), letters.size, N.ptr(off),
                                                                        len(off) - 1, 0, out, cap, found, N.ALGO_FILTER, 1), want)
    bits, n_bits = pkg.automaton._word_bits(("bytes", b"aAbB"), 1)
    kept = R.expand(R.words(hays, R.reps(letters, off), set(b"aAbB").__contains__))
    assert 0 < len(kept) < len(want)
    check_host_capacities(lambda out, cap, found: N.lib().acb_scan_host_words(
        tb, N.ptr(letters), letters.size, N.ptr(off), len(off) - 1, 0, N.ptr(bits), n_bits, out, cap, found,
        N.ALGO_FILTER, 1), kept)
    wide = [h + [0x2D] * (600 - len(h)) for h in hays] * 4
    d = torch.from_numpy(np.array(wide, dtype=np.uint8)).cuda()
    dl = np.array(wide, dtype=np.uint8).reshape(-1)
    want = R.find_all(dl, np.arange(len(wide) + 1, dtype=np.int64) * 600)
    assert len(want) > 4096
    A._match_cap = 0
    _same(rows(A.find_all_batch(d, ascii_case_insensitive=True)), want, "device route")
    assert A._match_cap > 4096


# ------------------------------------------------------------------ GPU: 6. sort keys of 64 and 65 bits with groups
def bits_for(v):
    b = 1
    while b < 64 and v >> b:
        b += 1
    return b


def _long_key_case(log_len, rng):
    """32 MiB in 2^18 haystacks of mixed-case text; keys: one of 2^log_len letters (it never matches; it sets the
    length field of the sort key), short keys that end together and case variants of them (groups of 2..4)"""
    short = [b"wxyz", b"xyz", b"yz", b"zz", b"qwxy"]
    keys = [tuple(k) for k in short] + [tuple(b"WXYZ"), tuple(b"XyZ"), tuple(b"xYz"), tuple(b"YZ"), tuple(b"Zz")]
    keys.append(tuple(rng.choice(np.frombuffer(b"abcd", dtype=np.uint8), size=1 << log_len).tolist()))
    n = 32 * MiB
    flat = rng.choice(np.frombuffer(b"efghijklmnop", dtype=np.uint8), size=n)
    for i, b in enumerate(range(50, n - 8, 1031)):
        k = short[i % 4] if i % 3 else b"qwxyz"
        flat[b:b + len(k)] = mixcase(np.frombuffer(k, dtype=np.uint8), rng)
    off = np.concatenate([[0], np.sort(rng.integers(0, n, size=(1 << 18) - 1)), [n]]).astype(np.int64)
    return keys, flat, off


def _by_key_id_last(r, kl):
    """the records in the reference order with key id as the last key"""
    return r[np.lexsort((r[:, 2], -kl[r[:, 2]], r[:, 1], r[:, 0]))]


@pytest.mark.gpu
@pytest.mark.parametrize("log_len", [19, 20])
def test_gpu_sort_key_width_with_groups(log_len, monkeypatch):
    """64 bits (2^19 letters): the host route sorts on the device; 65 bits (2^20): on the host (RefOrder).  The device
    tensor route with its device sort, and with the device sort refusing (np.lexsort).  Every group adjacent and in
    ascending key id, as the reference and a lexsort with key id last order them."""
    import torch
    rng = np.random.default_rng(log_len)
    keys, flat, off = _long_key_case(log_len, rng)
    assert bits_for(len(off) - 2) + bits_for(flat.size) + bits_for(1 << log_len) == (64 if log_len == 19 else 65)
    A = build("bytes", keys)
    R = Ref(keys, 1)
    want = R.find_all(flat, off)
    assert len(want) > 50_000 and np.array_equal(_by_key_id_last(want, R.kl), want)
    assert len(want) > len(R.reps(flat, off)) + 10_000
    A._match_cap = len(want) + 1024
    A.find_all_batch((flat, off), ascii_case_insensitive=True)         # every workspace grown (the expansion's too)
    count, m = launches(lambda: A.find_all_batch((flat, off), ascii_case_insensitive=True))
    assert count == 4 + (log_len == 19)                                # fold, scan, expansion, and the device sort at 64 bits
    _same(rows(m), want, "host route")
    rows2d = flat[:(flat.size // 4096) * 4096].reshape(-1, 4096)[:2000]
    d = torch.from_numpy(np.ascontiguousarray(rows2d)).cuda()
    dwant = R.find_all(rows2d.reshape(-1), np.arange(len(rows2d) + 1, dtype=np.int64) * 4096)
    _same(rows(A.find_all_batch(d, ascii_case_insensitive=True)), dwant, "device route, device sort")
    calls = []

    def refuse(*a):
        calls.append(a[2])
        return N.ACB_ERANGE
    monkeypatch.setattr(N.lib(), "acb_sort_matches_device", refuse)
    got = rows(A.find_all_batch(d, ascii_case_insensitive=True))
    assert calls == [len(dwant)]
    _same(got, dwant, "device route, host lexsort")
    assert np.array_equal(_by_key_id_last(got, R.kl), got)


# ------------------------------------------------------------------ GPU: 7. past 2 GiB
BIG_KEYS = [b"qvxjyk", b"wymbrp", b"hgfdsl", b"ntcuoe", b"ikaqwy", b"plokmj", b"zzzzzz"]     # z only in the last


def _big_text(n, plants, rng):
    """n bytes of '-' with the keys planted at (start, key index), each in random case"""
    t = np.full(n, 0x2D, dtype=np.uint8)
    for st, j in plants:
        k = np.frombuffer(BIG_KEYS[j], dtype=np.uint8)
        t[st:st + len(k)] = mixcase(k, rng)
    return t


def _by_construction(plants, off, R):
    """the records of the plants that lie inside one haystack, every alias after its representative"""
    out = []
    for st, j in plants:
        h = int(np.searchsorted(off, st, side="right")) - 1
        e = st + 6 - 1
        if off[h] <= st and e < off[h + 1]:
            out.append((h, e - off[h], j))
    out.sort()
    return R.expand(np.array(out, dtype=np.int64).reshape(-1, 3))


def _oracle_windows(t, off, got, R, at):
    """the records ending in [x - 300, x + 300) of the haystack holding x, against the oracle over that folded window"""
    for x in at:
        h = int(np.searchsorted(off, x, side="right")) - 1
        a, b = max(off[h], x - 300), min(off[h + 1], x + 300)
        if a >= b:
            continue
        w = R.find_all(t[a:b], np.array([0, b - a], dtype=np.int64))
        w[:, 0], w[:, 1] = h, w[:, 1] + a - off[h]
        sel = got[(got[:, 0] == h) & (got[:, 1] + off[h] >= a + 5) & (got[:, 1] + off[h] < b)]
        _same(sel, w, f"window at {x}")


@pytest.mark.gpu
def test_gpu_past_2_gib():
    """Keys in mixed case at row and haystack edges, either side of byte 2^31 (the second scan segment's first byte) and
    every few MiB.  A CUDA tensor of 525 rows of 4 MiB + 48 (2.2 GB: the folded copy passes 2^31 bytes, two scan
    segments; case variants, so the expansion runs); then a 2.2 GB host batch without variants (the pipeline, three
    launches per chunk) and with them (one piece: the batch and its folded copy both past 2 GiB).  Checked by
    construction and against the oracle in windows around the edges.  Device memory in use, measured on one H100 80GB
    HBM3: 5.7 GB after the tensor scan, 6.2 GB at most after the host scans (batch and folded copy); the host holds the
    2.2 GB text and, while the tensor is made, one copy more."""
    import torch
    rng = np.random.default_rng(31)
    G = 1 << 31
    stride, n_rows = 4 * MiB + 48, 525
    n = stride * n_rows
    assert n > G + 48 * MiB
    r31 = G // stride
    plants = []
    for r in range(n_rows):
        plants += [(r * stride, r % 6), ((r + 1) * stride - 6, (r + 1) % 6), (r * stride + 1 * MiB + r, (r + 2) % 6)]
    plants += [(G - 6 + i, 6) for i in range(7)]                       # twelve z: zzzzzz ends at 2^31 - 1, starts at 2^31,
    plants += [(G - 40, 4), (G + 40, 5)]                                # and crosses it at every offset
    plants = sorted(set(plants))
    assert all(b[0] >= a[0] + 6 or a[1] == b[1] == 6 for a, b in zip(plants, plants[1:]))
    t = _big_text(n, plants, rng)
    variants = [tuple(k) for k in BIG_KEYS] + [swap(tuple(k)) for k in BIG_KEYS[:3]] + \
        [tuple(k[:3].upper() + k[3:]) for k in BIG_KEYS[:2]] + [tuple(b"zzzZZZ")]
    edges = [G, G - 1, G + 1, r31 * stride, (r31 + 1) * stride]
    # the CUDA tensor
    A = build("bytes", variants)
    R = Ref(variants, 1)
    off = np.arange(n_rows + 1, dtype=np.int64) * stride
    want = _by_construction(plants, off, R)
    d = torch.from_numpy(t.reshape(n_rows, stride)).cuda()
    got = rows(A.find_all_batch(d, ascii_case_insensitive=True))
    peak = [used()]
    _same(got, want, "tensor")
    _oracle_windows(t, off, got, R, edges)
    for r in (0, r31, n_rows - 1):                                      # whole rows against the oracle
        w = R.find_all(t[r * stride:(r + 1) * stride], np.array([0, stride], dtype=np.int64))
        w[:, 0] = r
        _same(got[got[:, 0] == r], w, f"row {r}")
    assert np.array_equal(d[r31 - 1:r31 + 2].cpu().numpy().reshape(-1), t[(r31 - 1) * stride:(r31 + 2) * stride])
    del d
    torch.cuda.empty_cache()
    # the host batch, ragged, with haystack edges on plants' first and last bytes
    cuts = np.sort(np.concatenate([rng.integers(0, n, size=800), [G, G, G - 3, G + 4],
                                   [p[0] for p in plants[::50]], [p[0] + 6 for p in plants[25::50]]]))
    off = np.concatenate([[0], cuts, [n]]).astype(np.int64)
    nch = -(-n // CHUNK)
    for with_variants in (False, True):
        ks = variants if with_variants else [tuple(k) for k in BIG_KEYS]
        A = build("bytes", ks)
        R = Ref(ks, 1)
        want = _by_construction(plants, off, R)
        A._match_cap = len(want) + 1024
        A.find_all_batch((t, off), ascii_case_insensitive=True)         # every workspace grown
        count, m = launches(lambda: A.find_all_batch((t, off), ascii_case_insensitive=True))
        peak.append(used())
        assert count == (1 + 2 + 2 + 1 if with_variants else 3 * nch), count     # fold, 2 segments, expansion, sort
        got = rows(m)
        _same(got, want, f"host batch, variants={with_variants}")
        _oracle_windows(t, off, got, R, edges + [c * CHUNK for c in (64, 65)] + list(cuts[::97]))
        del A, m
        torch.cuda.empty_cache()
    print(f"device memory in use after each scan: {[round(x / 1e9, 2) for x in peak]} GB")


def used():
    import torch
    free, total = torch.cuda.mem_get_info()
    return total - free
