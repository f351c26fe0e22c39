"""Forced filter shapes of the scan kernels, their key sets and texts, shared by test_kernel_matrix.py,
test_record_bounds.py and test_stream_scale.py.  Not a test module.

A cell forces its shape (ACB_FILTER=g,s,log1,mode and ACB_FORCE_TAGMAP, only around make_automaton) on a key set whose
shortest key is exactly gram + stride - one letter; _check_shape reads it back with filter_shape()."""
import dataclasses

import numpy as np

import emul
import pyahocorasick_b200 as ac

RUN = 32                          # kLaneBytes: one lane's bytes per slice
SLICE = 32 * RUN                  # kSliceBytes: one consumer warp's slice
TILE = 20 * SLICE                 # kTileBytes (ACB_TILE_SLICES slices)
MiB = 1 << 20


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


def _big_batch(rng, keys, n):
    """n bytes of text in no key's letters with keys planted every few KiB, cut into a ragged batch"""
    flat = rng.choice(np.frombuffer(b"#%&*+-", dtype=np.uint8), size=n)
    for i, b in enumerate(range(100, n - 64, 4093)):
        k = keys[i % len(keys)]
        flat[b:b + len(k)] = np.frombuffer(k, dtype=np.uint8)
    cuts = np.sort(rng.integers(0, n, size=600))
    off = np.concatenate([[0, 0], cuts, [32 * MiB] * 3, [n, n]]).astype(np.int64)
    return flat, np.sort(off)
