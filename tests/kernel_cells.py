"""Forced filter shapes of the scan kernels, their key sets and texts, the kernels' ring geometry and the oracle
comparison, shared by test_kernel_matrix.py, test_scan_ring.py, test_record_bounds.py and test_stream_scale.py.  Not a
test module.

A cell forces its shape (ACB_FILTER=g,s,log1,mode and ACB_FORCE_TAGMAP, only around make_automaton) on a key set whose
shortest key is exactly gram + stride - one letter; _check_shape reads it back with filter_shape().  The tile a cell's
text is planted at is the tile of the kernel the cell runs, as the library reports it (acb_scan_geometry)."""
import collections
import ctypes
import dataclasses
import functools

import numpy as np
import pytest

import emul
import oracle
import pyahocorasick_b200 as ac
from pyahocorasick_b200 import _native as N
from batch_cases import triples

RUN = 32                          # kLaneBytes: one lane's bytes per slice
SLICE = 32 * RUN                  # kSliceBytes: one consumer warp's slice (the pair kernel static-asserts 1 KiB)
MiB = 1 << 20


# ------------------------------------------------------------------ the kernels' tile rings
Ring = collections.namedtuple("Ring", "slice tile stages consumers claim_depth look")


@functools.lru_cache(maxsize=None)
def geometry(pair):
    """the tile ring of acb_pair_kernel (pair) or acb_stream_kernel, from the constants the library was compiled with"""
    out = (ctypes.c_int32 * 6)()
    N.check(N.lib().acb_scan_geometry(int(bool(pair)), out, 6))
    return Ring(*out)


def sentinels(ring):
    """the fills the producer hands out when its claims run dry: one slice for every consumer warp"""
    slices = ring.tile // ring.slice
    return (ring.consumers + slices - 1) // slices


def tile_bytes(cell):
    """the tile of the kernel this cell runs on"""
    return geometry(cell.pair).tile


@dataclasses.dataclass(frozen=True)
class Cell:
    L: int                        # letter bytes: 1 bytes, 2 bytes-flavour KEY_SEQUENCE, 4 unicode
    g: int                        # gram bytes
    s: int                        # probe stride in bytes
    log1: int = 0                 # level-1 bitmap of 2^log1 bits; 0: the cost model's
    pair: bool = False
    tagmap: bool = False

    @property
    def env(self):
        return f"{self.g},{self.s},{self.log1},{int(self.pair)}"

    @property
    def name(self):
        kind = "pair" if self.pair else f"L{self.L}-g{self.g}-s{self.s}"
        return kind + (f"-l{self.log1}" if self.log1 else "") + ("-tag" if self.tagmap else "")


# ------------------------------------------------------------------ the cells: every instantiation
STRIDES = (1, 2, 4, 8, 16)
PAIR_LOG1 = (13, 16, 19, 20)      # level 2 of 2^13 / 2^16 / 2^19 bits (acb_pair_kernel<0>), 2^17 (acb_pair_kernel<17>)
GRAMS = {1: range(1, 17), 2: range(2, 17, 2), 4: range(4, 17, 4)}      # a gram is whole letters, at most 16 bytes


def _cells():
    """The shapes the dispatcher accepts: a stride of L * 2^k <= 16 bytes, a gram of whole letters up to 16 bytes, the
    pair placement only for 1-byte letters at gram 4 / stride 1; level 1 and the tag bitmap on a spread of them."""
    stream = [Cell(L, g, s) for L in (1, 2, 4) for g in GRAMS[L] for s in STRIDES if s >= L]
    pair = [Cell(1, 4, 1, log1, True, tag) for log1 in PAIR_LOG1 for tag in (False, True)]
    spread = ([dataclasses.replace(c, log1=13) for c in stream[0::9]] +       # saturated level 1
              [dataclasses.replace(c, log1=20) for c in stream[3::9]] +
              [dataclasses.replace(c, tagmap=True) for c in stream[6::9]])
    return stream + pair + spread


CELLS = _cells()
IDS = [c.name for c in CELLS]


def all_instantiations():
    modes = ("narrow", "wide")
    return ({("stream", nw, s, m) for nw in range(1, 5) for s in STRIDES for m in modes} |
            {("pair", 0), ("pair", 17), ("pair-tagmap",)})


def instantiation(fs):
    """the kernel template a scan with these tables launches (launch_stream / launch_pair)"""
    if fs["filter_flags"] & emul.FILTER_PAIR:
        return ("pair", 17 if fs["log2_bits2"] == 17 else 0)
    return ("stream", (fs["gram_bytes"] + 3) // 4, fs["stride"], "wide" if fs["filter_flags"] & emul.FILTER_WIDE else "narrow")


def cell_instantiation(cell):
    """the instantiation a cell forces, without building it (the pair cells with the tag bitmap count for it)"""
    if cell.pair:
        return ("pair-tagmap",) if cell.tagmap else ("pair", 17 if cell.log1 >= 20 else 0)
    return ("stream", (cell.g + 3) // 4, cell.s, "wide" if cell.g % 4 == 0 else "narrow")


# ------------------------------------------------------------------ key sets and text, in letters
ALPHA = {1: [0x61, 0x62, 0x63], 2: [0x0061, 0x6162, 0xFFFF], 4: [0x61, 0x142, 0x1F600]}
TOP = {1: 0xFF, 2: 0xFFFF, 4: 0x10FFFF}          # the largest letter; 0 is the smallest (the zero fill past the end)


def _keys(cell, rng):
    """Keys of at least m = (g + s - L) / L letters, at least one of exactly m: the forced gram is then the longest this
    key set offers at the forced stride."""
    L, alpha = cell.L, ALPHA[cell.L]
    m, gl, sl = (cell.g + cell.s - L) // L, cell.g // L, cell.s // L
    keys = []

    def rnd(n):
        return tuple(int(x) for x in rng.choice(alpha, size=n))

    def add(k):
        if len(k) >= m:
            keys.append(tuple(k))

    for _ in range(24):                                         # random keys, most longer than the 20 bytes an entry holds
        add(rnd(int(rng.integers(m, m + 24 // L + 4))))
    grm = rnd(gl)                                               # one gram at every probe offset j: anchor chains of one tag
    for j in range(sl):
        for _ in range(2):
            add(rnd(j) + grm + rnd(max(0, m - j - gl) + int(rng.integers(0, 4))))
    pre = rnd(gl + 3)                                           # a prefix longer than the gram: MULTI entries, trie walks
    for _ in range(5):
        add(pre + rnd(max(0, m - len(pre)) + int(rng.integers(0, 6))))
    for nb in (70, 100):                                        # longer than the DFA's 64-byte warm-up span
        add(rnd(max(m, nb // L)))
    k = rnd(m + 3)                                              # nested prefixes and suffixes: order inside one end index
    for x in (k, k + rnd(2), rnd(1) + k, k[1:], k[:m], rnd(2) + k + rnd(1), k[2:]):
        add(x)
    x, y = alpha[0], alpha[1]                                   # periodic keys: alternating text is all hits
    for n in (m, m + 1, m + 5):
        add(((x, y) * n)[:n])
        add(((y, x) * n)[:n])
    add(rnd(m) + (0, 0))                                        # against the zero fill of the last tile
    add((0,) * m)
    add((TOP[L],) * 2 + rnd(m))
    if L == 4:                                                  # no key for the latin-1 automaton (it ignores ACB_FILTER)
        keys = [k if max(k) > 0xFF else (0x142,) + k[1:] for k in keys]
    keys = list(dict.fromkeys(keys))
    assert min(map(len, keys)) == m
    return keys


def _pkg_key(k, L):
    if L == 1:
        return bytes(k)
    if L == 2:
        return k
    return "".join(map(chr, k))


def _build(cell, keys, mp):
    mod = ac.flavour("unicode" if cell.L == 4 else "bytes")
    A = mod.Automaton(mod.STORE_INTS, mod.KEY_SEQUENCE) if cell.L == 2 else mod.Automaton(mod.STORE_INTS)
    for i, k in enumerate(keys):
        A.add_word(_pkg_key(k, cell.L), i)
    with mp.context() as m:
        m.setenv("ACB_FILTER", cell.env)
        if cell.tagmap:
            m.setenv("ACB_FORCE_TAGMAP", "1")
        else:
            m.delenv("ACB_FORCE_TAGMAP", raising=False)
        A.make_automaton()
    return A


def _check_shape(A, cell):
    fs = A.filter_shape()
    assert (fs["gram_bytes"], fs["stride"]) == (cell.g, cell.s), fs
    if cell.pair:
        assert fs["filter_flags"] == emul.FILTER_PAIR and fs["log2_bits2"] == (17 if cell.log1 >= 20 else cell.log1), fs
    else:
        assert fs["filter_flags"] == (emul.FILTER_WIDE if cell.g % 4 == 0 else 0) and fs["log2_bits2"] == 0, fs
    if cell.log1:
        assert fs["log2_bits1"] == cell.log1, fs
    if cell.tagmap:
        assert fs["log2_bits3"] >= 16, fs
    elif cell.pair:
        assert fs["log2_bits3"] == 0, fs
    return fs


def _dense(cell, n_bytes):
    """alternating letters: every probe's gram belongs to a periodic key, so every probe of a slice is pending and a
    match ends at nearly every letter (item-list split, full candidate lists, match staging overflow)"""
    x, y = ALPHA[cell.L][:2]
    return np.array([x, y] * (n_bytes // cell.L // 2) + [x], dtype=np.uint32)


def _seed(cell):
    return sum(cell.name.encode()) * 7919 + cell.L


def _text(cell, keys, rng, n_bytes):
    """n_bytes of text in the key alphabet (a few 0 and top letters), keys planted across every lane-run, slice and tile
    boundary of the cell's kernel (coarser boundaries last, so that their keys survive) at every residue of the stride,
    and one key ending on the last byte.  Returns the letters and the start letters of the boundary plants."""
    L = cell.L
    n = n_bytes // L
    t = rng.choice(ALPHA[L], size=n).astype(np.uint32)
    odd = rng.random(n)
    t[odd < 0.01] = 0
    t[odd > 0.99] = TOP[L]
    plant = [k for k in keys if len(k) >= 2]
    starts, i = [], 0
    for step in (RUN, SLICE, tile_bytes(cell)):
        for b in range(step, n_bytes, step):
            k = plant[(i * 7) % len(plant)]
            d = 1 + (i >> 1) % (cell.s // L) if i % 2 == 0 else 1 + (i * 5) % (len(k) - 1)    # letters before b
            st = b // L - d
            if 0 <= st and st + len(k) <= n:
                t[st:st + len(k)] = k
                starts.append(st)
            i += 1
    k = plant[i % len(plant)]
    t[n - len(k):] = k
    return t, np.asarray(starts, dtype=np.int64)


def _ragged(rng, n, starts, boundaries):
    """offsets (in letters) of a ragged batch over n letters: random cuts, cuts through planted keys and at tile
    boundaries, runs of empty haystacks, empty haystacks first and last"""
    cuts = [rng.integers(0, n + 1, size=120), starts[rng.integers(0, len(starts), size=80)] + 1, boundaries]
    cuts = np.sort(np.concatenate(cuts))
    cuts = np.concatenate([cuts, cuts[::17], cuts[::17], cuts[5::23]])           # repeated offsets: empty haystacks
    return np.concatenate([[0, 0], np.sort(np.clip(cuts, 0, n)), [n, n]]).astype(np.int64)


def _big_batch(rng, keys, n):
    """n bytes of text in no key's letters with keys planted every few KiB, cut into a ragged batch"""
    flat = rng.choice(np.frombuffer(b"#%&*+-", dtype=np.uint8), size=n)
    for i, b in enumerate(range(100, n - 64, 4093)):
        k = keys[i % len(keys)]
        flat[b:b + len(k)] = np.frombuffer(k, dtype=np.uint8)
    cuts = np.sort(rng.integers(0, n, size=600))
    off = np.concatenate([[0, 0], cuts, [32 * MiB] * 3, [n, n]]).astype(np.int64)
    return flat, np.sort(off)


# ------------------------------------------------------------------ the oracle
def _oracle_key(k, L):
    return bytes(k) if L == 1 else k


def _oracle(cell, keys):
    O = oracle.OracleAutomaton()
    for i, k in enumerate(keys):
        O.add_word(_oracle_key(k, cell.L), i)
    O.make_automaton()
    return O


def _want(O, cell, letters, off):
    if cell.L == 1:
        return [tuple(r) for r in O.scan_batch_bytes(letters.astype(np.uint8), off).tolist()]
    return O.scan_batch_letters(letters, off)


def _diff(got, want):
    """a short account of how two record lists differ (the first divergence, a few missing and extra records)"""
    i = next((i for i, (a, b) in enumerate(zip(got, want)) if a != b), min(len(got), len(want)))
    sg, sw = set(got), set(want)
    return (f"{len(got)} records, want {len(want)}; first difference at {i}: got {got[i:i + 3]}, want {want[i:i + 3]}; "
            f"missing {sorted(sw - sg)[:5]}, extra {sorted(sg - sw)[:5]}")


def _check_gpu(A, batch, want, what, dfa=True):
    """filter (and DFA) records equal the oracle's in order; unsorted filter records equal them as a set"""
    for algo in ("filter", "dfa") if dfa else ("filter",):
        got = triples(A.find_all_batch(batch, algo=algo))
        if got != want:
            pytest.fail(f"{what}, {algo}: {_diff(got, want)}")
    got = sorted(triples(A.find_all_batch(batch, algo="filter", sort=False)))
    if got != sorted(want):
        pytest.fail(f"{what}, filter unsorted: {_diff(got, sorted(want))}")
