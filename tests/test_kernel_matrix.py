"""Every compiled scan kernel against the C oracle, one cell per filter shape.

acb_stream_kernel<NW, STRIDE, MODE> is compiled 40 times (NW = 1..4 hash windows for grams of 1..16 bytes, STRIDE
1..16, MODE wide iff the gram is a multiple of 4 bytes) and acb_pair_kernel<L2B> twice (a level 2 of 2^17 bits or any
other size).  Each has its own unrolled probe loop, last-slice mask, item-list split and anchor offsets, and which one
a scan runs on follows from the key set (build_filter's cost model).  So every cell here forces its shape
(ACB_FILTER=g,s,log1,mode and ACB_FORCE_TAGMAP, only around make_automaton) on a key set whose shortest key is exactly
gram + stride - one letter, checks with filter_shape() that the forcing took, and compares with the oracle:

  GPU (-m gpu)  the filter and the DFA kernels on three tiles of the cell's kernel (as acb_scan_geometry reports its
                ring) plus a ragged tail, with keys planted across every 32-byte lane run, 1 KiB slice and tile boundary and at every residue of the stride; the same bytes as a
                ragged batch (empty haystacks, cuts through planted keys) and at two fixed strides; and text on which
                every probe is a hit.  Records must equal the oracle's in order; unsorted, as a set.
  CPU           the same forced tables through tests/emul.py (the kernels restated in Python) on about 2 KiB, so that
                a failing GPU cell shows whether the tables or the kernel are wrong.

The coverage tests read the shapes back and require all 42 instantiations plus the pair kernel with the tag bitmap.
"""
import numpy as np
import pytest

import emul
import pyahocorasick_b200 as ac
from batch_cases import DT, triples
from kernel_cells import (CELLS, IDS, SLICE, Cell, _build, _check_gpu, _check_shape, _dense, _diff, _keys, _oracle, _ragged,
                          _seed, _text, _want, all_instantiations, instantiation, tile_bytes)


# ------------------------------------------------------------------ GPU: the kernels
_RAN = set()                  # instantiations that went through a whole GPU cell


@pytest.mark.gpu
@pytest.mark.parametrize("cell", CELLS, ids=IDS)
def test_kernel_cell_matches_oracle(cell, monkeypatch):
    rng = np.random.Generator(np.random.PCG64(_seed(cell)))
    keys = _keys(cell, rng)
    A = _build(cell, keys, monkeypatch)
    fs = _check_shape(A, cell)
    O = _oracle(cell, keys)
    L, dt = cell.L, DT[cell.L]
    tile = tile_bytes(cell)
    n_bytes = 3 * tile + L * 1291                     # a ragged tail: not a multiple of 16, nor of a stride above L
    t, starts = _text(cell, keys, rng, n_bytes)
    n = t.size
    flat = t.astype(dt).view(np.uint8)
    # 1. one haystack
    one = np.array([0, n], dtype=np.int64)
    want = _want(O, cell, t, one)
    assert len(want) > len(starts) // 2                # most plants survive the ones planted over them
    _check_gpu(A, (flat, one * L), want, "one haystack")
    # 2. ragged, with empty haystacks and cuts through planted keys
    roff = _ragged(rng, n, starts, np.arange(tile // L, n, tile // L))
    _check_gpu(A, (flat, roff * L), _want(O, cell, t, roff), "ragged batch")
    # 3. fixed strides: a power of two (shift) and not (division)
    for stride in (512, 3000):
        k = flat.size // stride
        foff = np.arange(k + 1, dtype=np.int64) * (stride // L)
        _check_gpu(A, flat[:k * stride].reshape(k, stride), _want(O, cell, t[:k * (stride // L)], foff), f"stride {stride}")
    # 4. every probe a hit
    d = _dense(cell, tile + 3 * SLICE)
    doff = np.array([0, d.size], dtype=np.int64)
    dwant = _want(O, cell, d, doff)
    assert len(dwant) > 2 * d.size                     # several periodic keys end at every letter
    _check_gpu(A, (d.astype(dt).view(np.uint8), doff * L), dwant, "dense text")
    _RAN.add(instantiation(fs))
    if cell.pair and fs["log2_bits3"]:
        _RAN.add(("pair-tagmap",))


@pytest.mark.gpu
def test_every_kernel_instantiation_ran(request):
    """the cells above, as they ran on the GPU, reached every instantiation (run after them, in one session)"""
    names = {it.name for it in request.session.items}
    if not all(f"test_kernel_cell_matches_oracle[{i}]" in names for i in IDS):
        pytest.skip("only part of the kernel matrix was selected")
    assert _RAN == all_instantiations(), sorted(all_instantiations() - _RAN, key=str)


# ------------------------------------------------------------------ CPU: the forced tables
def test_cells_reach_every_kernel_instantiation(monkeypatch):
    """the cells' tables, as filter_shape() reports them, select all 40 stream and 2 pair instantiations, and the pair
    kernel with the tag bitmap; adding an instantiation or dropping a cell fails here"""
    seen = set()
    for cell in CELLS:
        A = _build(cell, _keys(cell, np.random.Generator(np.random.PCG64(_seed(cell)))), monkeypatch)
        fs = _check_shape(A, cell)
        seen.add(instantiation(fs))
        if cell.pair and fs["log2_bits3"]:
            seen.add(("pair-tagmap",))
    assert seen == all_instantiations(), sorted(all_instantiations() ^ seen, key=str)


@pytest.mark.parametrize("cell", CELLS, ids=IDS)
def test_cell_tables_match_oracle_emulated(cell, monkeypatch):
    rng = np.random.Generator(np.random.PCG64(_seed(cell)))
    keys = _keys(cell, rng)
    A = _build(cell, keys, monkeypatch)
    _check_shape(A, cell)
    f = A.flat()
    O = _oracle(cell, keys)
    L, dt = cell.L, DT[cell.L]
    t, starts = _text(cell, keys, rng, 2048 + L * 53)
    n = t.size
    flat = t.astype(dt).view(np.uint8)
    d = _dense(cell, 160)
    layouts = [("one haystack", t, np.array([0, n], dtype=np.int64)),
               ("ragged batch", t, _ragged(rng, n, starts, np.arange(SLICE // L, n, SLICE // L))),
               ("dense text", d, np.array([0, d.size], dtype=np.int64))]
    for what, letters, off in layouts:
        want = _want(O, cell, letters, off)
        buf = flat if letters is t else letters.astype(dt).view(np.uint8)
        for name, fn in (("filter", emul.emul_filter), ("dfa", emul.emul_dfa)):
            got = fn(f, buf, off * L, 0)
            if got != want:
                pytest.fail(f"{what}, emulated {name}: {_diff(got, want)}")


# ------------------------------------------------------------------ the forcing hook refuses what no kernel can run
def _forced(monkeypatch, env, keys, flavour="bytes"):
    mod = ac.flavour(flavour)
    A = mod.Automaton(mod.STORE_INTS, mod.KEY_SEQUENCE) if isinstance(keys[0], tuple) else mod.Automaton(mod.STORE_INTS)
    for i, k in enumerate(keys):
        A.add_word(k, i)
    with monkeypatch.context() as m:
        m.setenv("ACB_FILTER", env)
        A.make_automaton()
    return A


EIGHT = [b"abcdefgh", b"abcdefgx", b"bcdefghijk"]


@pytest.mark.parametrize("env, flavour, keys, msg", [
    ("16,16,0,0", "bytes", EIGHT, "not a candidate"),             # g + s would need keys of 31 bytes
    ("8,2,0,0", "bytes", EIGHT, "not a candidate"),               # at stride 2 the grams stop at 7 bytes
    ("6,1,0,0", "bytes", EIGHT, "not a candidate"),               # neither gmax (8) nor 4
    ("0,0,0,0", "bytes", [b"a", b"ab"], None),                    # nothing forced: allowed
    ("4,3,0,0", "bytes", EIGHT, "stride"),
    ("4,32,0,0", "bytes", EIGHT, "stride"),
    ("4,1,0,0", "bytes", [(1, 2, 3, 4), (5, 6, 7, 8)], "stride"),    # 2-byte letters: a stride of 1 byte is no letter
    ("8,2,0,0", "unicode", ["łabcdefgh"], "stride"),
    ("3,2,0,0", "bytes", [(1, 2, 3, 4), (5, 6, 7, 8)], "gram"),      # half a letter
    ("4,1,22,0", "bytes", EIGHT, "log1"),                         # 2^22 bits: no room in shared memory
    ("4,1,12,0", "bytes", EIGHT, "log1"),
    ("8,1,0,1", "bytes", EIGHT, "pair"),
    ("4,2,0,1", "bytes", EIGHT, "pair"),
    ("0,0,0,1", "bytes", EIGHT, "pair"),
    ("4,2,0,1", "bytes", [(1, 2, 3, 4), (5, 6, 7, 8)], "pair"),
    ("4,1,0,2", "bytes", EIGHT, "mode"),
    ("x", "bytes", EIGHT, "expected"),
], ids=lambda v: v if isinstance(v, str) else None)
def test_infeasible_forced_shapes_are_refused(monkeypatch, env, flavour, keys, msg):
    if msg is None:
        assert _forced(monkeypatch, env, keys, flavour).kind == ac.AHOCORASICK
        return
    with pytest.raises(ValueError, match=msg):
        _forced(monkeypatch, env, keys, flavour)


def test_a_refused_forcing_leaves_a_trie_that_builds_without_it(monkeypatch):
    A = ac.flavour("bytes").Automaton(ac.STORE_INTS)
    for i, k in enumerate(EIGHT):
        A.add_word(k, i)
    with monkeypatch.context() as m:
        m.setenv("ACB_FILTER", "16,16,0,0")
        with pytest.raises(ValueError):
            A.make_automaton()
    assert A.kind == ac.TRIE
    with pytest.raises(AttributeError):
        A.filter_shape()
    monkeypatch.delenv("ACB_FILTER", raising=False)
    assert A.make_automaton() is None and A.kind == ac.AHOCORASICK
    fs = A.filter_shape()
    assert fs["gram_bytes"] + fs["stride"] - 1 <= 8 and fs["log2_bits1"] >= 13
    text = np.frombuffer(b"xxabcdefghx", dtype=np.uint8)
    assert emul.emul_filter(A.flat(), text, np.array([0, text.size], dtype=np.int64), 0) == [(0, 9, 0)]


# ------------------------------------------------------------------ the pipelined host scan on a ragged batch
MiB = 1 << 20
CHUNK = 32 * MiB                  # scan_host_pipelined's chunk; batches of 48 MiB and more take that path


@pytest.mark.gpu
@pytest.mark.parametrize("cell", [Cell(1, 7, 8), Cell(1, 4, 1, 16, True)], ids=lambda c: c.name)
def test_pipelined_scan_of_a_ragged_batch(cell, monkeypatch):
    """about 100 MiB in (flat, offsets) form: the host scan copies, scans and sorts it in 32 MiB chunks, a start
    position `reach` before a chunk boundary waits for the next chunk, and the runs of the haystacks a cut goes through
    are merged on the host.  Here one haystack spans three chunk sorts, haystack boundaries lie exactly on a chunk
    boundary and on a scan cut (the boundary minus the reach), and a run of empty haystacks sits on the chunk
    boundary.  The filter path (pipelined) must equal the oracle and the DFA path (one launch over the batch)."""
    rng = np.random.Generator(np.random.PCG64(_seed(cell)))
    keys = _keys(cell, rng)
    A = _build(cell, keys, monkeypatch)
    _check_shape(A, cell)
    reach = (max(map(len, keys)) + 31) & ~31
    n = 100 * MiB + 12345
    flat = rng.integers(ord("d"), ord("z") + 1, size=n, dtype=np.uint8)       # no key letter: the plants are the matches
    plant = [np.frombuffer(bytes(k), dtype=np.uint8) for k in keys]
    sites = list(range(4096, n - 256, 4093))
    for c in (1, 2, 3):                                                       # across every chunk boundary and scan cut
        for b in (c * CHUNK, c * CHUNK - reach):
            sites += [b - d for d in range(1, 2 * reach, 3)]
    for i, b in enumerate(sorted(sites)):
        k = plant[i % len(plant)]
        flat[b:b + len(k)] = k
    k = plant[0]
    flat[n - len(k):] = k
    long_hay = (10 * MiB, 80 * MiB)                                           # spans the cuts of chunks 1 and 2
    cuts = np.concatenate([[5 * MiB], rng.integers(5 * MiB, 10 * MiB, size=400), long_hay,
                           rng.integers(80 * MiB, 3 * CHUNK - reach, size=300),
                           [3 * CHUNK - reach] + [3 * CHUNK] * 5, rng.integers(3 * CHUNK + 1, n, size=200)])
    off = np.concatenate([[0], np.sort(cuts), [n]]).astype(np.int64)
    O = _oracle(cell, keys)
    want = _want(O, cell, flat, off)
    h_long = int(np.searchsorted(off, long_hay[0], side="right")) - 1
    ends = np.array([e + long_hay[0] for h, e, _ in want if h == h_long])
    assert off[h_long] == long_hay[0] and all(((ends >= a) & (ends < a + CHUNK)).any() for a in (0, CHUNK, 2 * CHUNK))
    for algo in ("filter", "dfa"):
        got = triples(A.find_all_batch((flat, off), algo=algo))
        if got != want:
            pytest.fail(f"{algo}: {_diff(got, want)}")
    got = sorted(triples(A.find_all_batch((flat, off), algo="filter", sort=False)))
    if got != sorted(want):
        pytest.fail(f"filter unsorted: {_diff(got, sorted(want))}")
