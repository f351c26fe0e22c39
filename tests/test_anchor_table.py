"""The anchor table's rare chains, built on purpose and walked on the GPU.

Every filter-path match ends in the anchor table, walked by three hand-written copies of one loop: resolve_chain
(inlined into every acb_stream_kernel), pair_resolve (foreign-tag skip, the single-entry fast path, one ballot and
atomic per warp turn) and pair_resolve_general.  Random key sets almost never reach their rare branches, so
tests/anchor_cases.py solves the tag hash for key sets that must: tags homed in the last slot whose chains wrap to slot
0, twin grams under one tag (UNIQUE + UNIQUE, UNIQUE + MULTI, MULTI + MULTI), one tag at two probe offsets, a tag's one
UNIQUE entry displaced by a foreign one, a tag behind eight foreign entries, MULTI entries of shared prefixes and long
keys, keys of 20 and 21 bytes.  Texts plant every key, near misses (the gram, another last letter) and decoys (a key
gram's tag, other bytes, shown to pass the bitmap) back to back and apart, at haystack starts and ends, across cuts
and on the buffer's last letters.

  CPU           per cell (every kernel_cells cell, plus unicode KEY_SEQUENCE cells): the table read back has every
                property the cell's shape allows, the decoys reach the walk, and the emulated kernels equal the oracle.
  GPU (-m gpu)  per cell the filter and DFA kernels against the oracle on one haystack, a ragged batch, a fixed stride
                and unsorted; for one pair cell and one wide stream cell a CUDA-tensor batch and a host batch over 48 MiB
                (the pipelined route, whose segments carry the same candidates at other offsets).
"""
import functools

import numpy as np
import pytest

import anchor_cases as ancs
import emul
import kernel_cells as kc
from anchor_cases import CELLS, IDS
from batch_cases import DT

MiB = 1 << 20


def _seed(c):
    return kc._seed(c.cell) * 3 + 17 * c.seq


def _oracle(c, keys):
    if not c.seq:
        return kc._oracle(c.cell, keys)
    import oracle
    O = oracle.OracleAutomaton()
    for i, k in enumerate(keys):
        O.add_word(tuple(k), i)
    O.make_automaton()
    return O


@functools.lru_cache(maxsize=None)
def _tables(c):
    """the plan, automaton and flat tables of a cell, built once per session (the CPU and GPU tests share them)"""
    with pytest.MonkeyPatch.context() as mp:
        plan, A, f = ancs.build(c, np.random.Generator(np.random.PCG64(_seed(c))), mp)
    if not c.seq:
        kc._check_shape(A, c.cell)
    return plan, A, f


def _setup(c, mp):
    """the cell's tables and a generator for its texts"""
    return (np.random.Generator(np.random.PCG64(_seed(c) + 1)),) + _tables(c)


def _decoys_reach_walk(c, f, plan, t, items):
    """every planted decoy passes the bitmaps at its probe position, and carries a tag some entry has"""
    buf = t.astype(DT[c.L]).view(np.uint8)
    tags = {e.tag for e in ancs.entries(f)}
    dec = [it for it in items if it.kind == "decoy"]
    for it in dec:
        q = it.start * c.L
        assert q % c.s == 0 and emul._passes_bitmap(f, buf, q), (c.name, it)
        assert emul.hash_bytes(buf, q, c.g, emul.multipliers(c.g, 2)) | 1 in tags
    return len(dec)


# ------------------------------------------------------------------ CPU: the tables and the emulated kernels
@pytest.mark.parametrize("c", CELLS, ids=IDS)
def test_table_has_the_chains(c, monkeypatch):
    """the built table has each property the cell's shape allows (named in the message when one is missing): a change
    to the hash or the table layout that stops the key set reaching a branch fails here"""
    _, plan, A, f = _setup(c, monkeypatch)
    have = ancs.properties(c, f, plan)
    want = ancs.capabilities(c)
    assert want <= have, f"{c.name}: missing {sorted(want - have)}; has {sorted(have)}"
    if ancs.has_twins(c):
        assert plan.decoys and all(ancs.tag_of(c, d) == t for d, t in plan.decoys)
    else:                                               # the tag is a bijection of the gram: no twins to find
        P = ancs._pool(c, np.random.Generator(np.random.PCG64(1)))
        if len(P) < 1 << 20:
            assert len(np.unique(ancs.tags(c, P))) == len(P)


@pytest.mark.parametrize("c", CELLS, ids=IDS)
def test_emulated_walk_matches_oracle(c, monkeypatch):
    rng, plan, A, f = _setup(c, monkeypatch)
    O = _oracle(c, plan.keys)
    z, items = ancs.zone(c, f, plan, rng)
    k = plan.keys[0]
    t = np.concatenate([z, np.asarray(k, dtype=np.int64)])
    items.append(ancs.Item(z.size, len(k), "key"))
    n = t.size
    assert (_decoys_reach_walk(c, f, plan, t, items) > 0) == bool(plan.decoys)
    buf = t.astype(DT[c.L]).view(np.uint8)
    for what, off in (("one haystack", np.array([0, n], dtype=np.int64)), ("ragged batch", ancs.ragged(c, rng, n, items))):
        want = kc._want(O, c.cell, t, off)
        for name, fn in (("filter", emul.emul_filter), ("dfa", emul.emul_dfa)):
            got = fn(f, buf, off * c.L, 0)
            if got != want:
                pytest.fail(f"{what}, emulated {name}: {kc._diff(got, want)}")


def test_every_property_is_reached(monkeypatch):
    """across the cells every construction shows up in some table (and the pair kernel meets twins and decoys)"""
    seen = set()
    for c in CELLS:
        if c.pair or c.seq or c.g in (1, 3):
            _, plan, A, f = _setup(c, monkeypatch)
            seen |= ancs.properties(c, f, plan)
    assert seen >= {"wrap", "wrap-split", "uu", "um", "mm", "two-j", "displaced", "run8", "shared", "long", "k20", "k21",
                    "one-tag"}, sorted(seen)


# ------------------------------------------------------------------ GPU: the kernels
@pytest.mark.gpu
@pytest.mark.parametrize("c", CELLS, ids=IDS)
def test_anchor_walk_matches_oracle(c, monkeypatch):
    rng, plan, A, f = _setup(c, monkeypatch)
    O = _oracle(c, plan.keys)
    L = c.L
    t, items = ancs.text(c, f, plan, rng, 2 * kc.tile_bytes(c.cell) + L * 1291)
    _decoys_reach_walk(c, f, plan, t, items)
    n = t.size
    flat = t.astype(DT[L]).view(np.uint8)
    one = np.array([0, n], dtype=np.int64)
    kc._check_gpu(A, (flat, one * L), kc._want(O, c.cell, t, one), "one haystack")
    roff = ancs.ragged(c, rng, n, items)
    kc._check_gpu(A, (flat, roff * L), kc._want(O, c.cell, t, roff), "ragged batch")
    stride = 3000
    k = flat.size // stride
    foff = np.arange(k + 1, dtype=np.int64) * (stride // L)
    kc._check_gpu(A, flat[:k * stride].reshape(k, stride), kc._want(O, c.cell, t[:k * (stride // L)], foff), f"stride {stride}")


BIG = [c for c in CELLS if (c.pair and c.log1 == 16 and not c.tagmap) or (c.name == "L1-g8-s4")]


@pytest.mark.gpu
@pytest.mark.parametrize("c", BIG, ids=[c.name for c in BIG])
def test_anchor_walk_device_and_pipelined_batches(c, monkeypatch):
    """a CUDA-tensor batch, and a host batch over 48 MiB: the pipelined route's segments start at other offsets of the
    same adversarial candidates"""
    import torch
    rng, plan, A, f = _setup(c, monkeypatch)
    O = _oracle(c, plan.keys)
    t, items = ancs.text(c, f, plan, rng, 2 * kc.tile_bytes(c.cell) + 1291)
    flat = t.astype(np.uint8)
    stride = 4096
    k = flat.size // stride
    foff = np.arange(k + 1, dtype=np.int64) * stride
    dev = torch.from_numpy(flat[:k * stride].reshape(k, stride).copy()).cuda()
    kc._check_gpu(A, dev, kc._want(O, c.cell, t[:k * stride], foff), "CUDA tensor")
    reps = (48 * MiB) // flat.size + 2
    big = np.tile(flat, reps)
    cuts = [ancs.ragged(c, rng, flat.size, items)[1:-1] + r * flat.size for r in range(0, reps, 7)]
    off = np.unique(np.concatenate([[0, big.size], rng.integers(0, big.size, size=3000)] + cuts)).astype(np.int64)
    off = np.concatenate([[0], off, [big.size]])
    assert big.size > 48 * MiB
    kc._check_gpu(A, (big, off), kc._want(O, c.cell, big, off), "48 MiB host batch", dfa=False)
