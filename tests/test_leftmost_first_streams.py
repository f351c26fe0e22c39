"""Leftmost-first stream batches (Automaton.stream_batch(leftmost_first=True), Replacer(leftmost_first=True).stream_batch)
and leftmost-first selection at the measured scale.

A stream's feeds and finish, concatenated, equal find_leftmost_first_batch / replace_batch of its whole text, and `re`
on it.  The CPU test runs the restatement of the feeds (tests/emul_leftmost_first.py) and checks after every feed what
has been reported and what is held; the gpu-marked tests run the real feeds and, at scale, the real selection against
the definition over find_all_batch's full list."""
import numpy as np
import pytest

import emul_leftmost_first as elf
import emul_words
import first_cases
from batch_cases import CASES, automaton, got_values, key_len, obj, oracle_full, replace_reps, rows

CHUNKS = [1, 7, 64, 256]


def _texts(rng, n, al, lo=0, hi=900):
    return [[int(x) for x in rng.choice(al, size=int(rng.integers(lo, hi)))] for _ in range(n)]


def _keys(rng, al, n=14):
    keys = [list(k) for k in {tuple(int(x) for x in rng.choice(al, size=int(rng.integers(1, 7)))) for _ in range(n)}]
    rng.shuffle(keys)
    return keys


# ------------------------------------------------------------------ the restatement (CPU)
@pytest.mark.parametrize("words", [False, True])
def test_restatement_reports_and_holds_what_it_must(words):
    """after every feed of chunks of 1, 7, 64, 256 and random sizes: every chosen match of the whole text that starts
    before P - T (words: P - T - 1) has been reported, nothing else has, at most T (T + 1) letters are held; after
    finish, everything, equal to `re` on the whole text"""
    rng = np.random.default_rng(31 + words)
    al = [0x61, 0x62, 0x20]
    for size in CHUNKS + [0]:
        keys = _keys(rng, al[:2])
        A, O = automaton("bytes", False, keys)
        kl = np.array([len(k) for k in keys])
        T = int(kl.max()) - 1
        H = T + int(words)
        hays = _texts(rng, 3, al)
        letters = [0x61] if words else None
        want = first_cases.find("bytes", keys, hays, letters)
        st = elf.new_state(A, len(hays), ("bytes", b"a") if words else None)
        got, pos = [], [0] * len(hays)
        while any(pos[h] < len(hays[h]) for h in range(len(hays))):
            ids = [h for h in range(len(hays)) if pos[h] < len(hays[h])]
            take = [size or int(rng.integers(1, 40)) for _ in ids]
            chunks = [bytes(hays[h][pos[h]:pos[h] + t]) for h, t in zip(ids, take)]
            got += [(ids[c], e + pos[ids[c]], k) for c, e, k in elf.feed(A.flat(), st, chunks, np.array(ids), "filter", False)]
            for h, t in zip(ids, take):
                pos[h] = min(pos[h] + t, len(hays[h]))
            for h in range(len(hays)):
                assert len(st["held"][h]) <= H
                settled = [r for r in want if r[0] == h and r[1] - kl[r[2]] + 1 < pos[h] - H]
                assert sorted(r for r in got if r[0] == h) == settled
        got += [(c, e + pos[c], k) for c, e, k in elf.feed(A.flat(), st, [b""] * len(hays), None, "filter", True)]
        assert sorted(got) == want
        assert all(not x for x in st["held"])
        full = oracle_full(O, hays)
        assert elf.greedy_first(emul_words.definition(hays, full, kl, lambda v: v == 0x61) if words else full, kl) == want


# ------------------------------------------------------------------ the real feeds
def _feed_all(B, texts, size, fl, seq, rng):
    """feed every stream in chunks of `size` letters (0: random sizes), some streams skipped in some feeds, then
    finish -> [(stream, end, value)] sorted"""
    got, pos = [], [0] * len(texts)
    while any(pos[s] < len(texts[s]) for s in range(len(texts))):
        ids = [s for s in range(len(texts)) if pos[s] < len(texts[s]) and rng.integers(0, 4)]
        if not ids:
            continue
        take = [size or int(rng.integers(1, 300)) for _ in ids]
        m = B.feed([obj(fl, seq, texts[s][pos[s]:pos[s] + t]) for s, t in zip(ids, take)], ids)
        got += got_values(m)
        for s, t in zip(ids, take):
            pos[s] = min(pos[s] + t, len(texts[s]))
    return sorted(got + got_values(B.finish()))


def _replace_all(RS, texts, size, fl, seq, rng):
    out = [[] for _ in texts]
    pos = [0] * len(texts)

    def add(items, ids):
        for s, x in zip(ids, items):
            out[s] += list(x) if not isinstance(x, str) else [ord(c) for c in x]
    while any(pos[s] < len(texts[s]) for s in range(len(texts))):
        ids = [s for s in range(len(texts)) if pos[s] < len(texts[s])]
        take = [size or int(rng.integers(1, 300)) for _ in ids]
        add(RS.feed([obj(fl, seq, texts[s][pos[s]:pos[s] + t]) for s, t in zip(ids, take)], ids), ids)
        for s, t in zip(ids, take):
            pos[s] = min(pos[s] + t, len(texts[s]))
    add(RS.finish(), range(len(texts)))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("size", CHUNKS + [0])
@pytest.mark.parametrize("case", ["bytes", "wide"])
def test_gpu_streams_equal_the_whole_text(case, size):
    fl, seq, al = CASES[case]
    rng = np.random.default_rng(size + (case == "wide"))
    al = al + [0x20]
    keys = _keys(rng, al[:2] + [0x20], 20)
    A, O = automaton(fl, seq, keys)
    texts = _texts(rng, 6, al, 0, 3000)
    word_letters = [c for c in al if c != 0x20]
    arg = bytes(word_letters) if fl == "bytes" else "".join(map(chr, word_letters))
    for whole, letters in ((False, None), (arg, word_letters)):
        want = first_cases.find(case, keys, texts, letters)
        whole_batch = got_values(A.find_leftmost_first_batch([obj(fl, seq, t) for t in texts], whole_words=whole))
        assert whole_batch == want
        B = A.stream_batch(len(texts), leftmost_first=True, whole_words=whole)
        assert _feed_all(B, texts, size, fl, seq, rng) == sorted(want), whole
        reps = replace_reps(case, keys, rng)
        R = A.replacer({obj(fl, seq, k): obj(fl, seq, r) for k, r in zip(keys, reps)}, leftmost_first=True)
        assert _replace_all(R.stream_batch(len(texts), whole_words=whole), texts, size, fl, seq, rng) == \
            first_cases.sub(case, keys, reps, texts, letters), whole


@pytest.mark.gpu
def test_gpu_stream_launch_counts():
    """a leftmost-first feed launches what a leftmost-longest feed launches (tests/test_stream_words.py pins those)"""
    from pyahocorasick_b200 import _native as N
    keys = [b"ab", b"abc", b"bc"]
    A, _ = automaton("bytes", False, [list(k) for k in keys])
    chunks = [b"ab abc bc " * 3, b"abc ab"]
    L = N.lib()

    def count(B):
        B.feed([b"a", b"b"])
        before = L.acb_launch_count()
        B.feed(chunks)
        return L.acb_launch_count() - before

    R = A.replacer({k: b"X" for k in keys}, leftmost_first=True)
    got = {"leftmost": count(A.stream_batch(2, leftmost_first=True)), "replace": count(R.stream_batch(2)),
           "leftmost_words": count(A.stream_batch(2, leftmost_first=True, whole_words=True)),
           "replace_words": count(R.stream_batch(2, whole_words=True))}
    assert got == {"leftmost": 14, "replace": 21, "leftmost_words": 15, "replace_words": 22}


# ------------------------------------------------------------------ scale
def _check_at_scale(A, batch):
    got = rows(A.find_leftmost_first_batch(batch))
    full = A.find_all_batch(batch)
    want = first_cases.np_greedy_first(np.rec.fromarrays([full.hay_id, full.end_index, full.key_id], names="hay_id,end_index,key_id"),
                                       key_len(A))
    assert np.array_equal(got, want)
    return got


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["C2", "C4"])
def test_gpu_at_scale(name):
    """C2 planted (1 M x 256 B) and C4 (64 x 16 MiB) under C2's 10 000 keys: the definition over find_all_batch's full
    list, with the keys in a shuffled order and added longest-first; added longest-first, leftmost-first is
    leftmost-longest record for record"""
    from pyahocorasick_b200 import synth
    w = synth.make(name)
    keys = list(w.keys)
    np.random.default_rng(3).shuffle(keys)
    A = synth.build_automaton(keys)
    got = _check_at_scale(A, w.haystacks)
    assert len(got) >= len(w.planted_hay)
    by_len = synth.build_automaton(sorted(w.keys, key=len, reverse=True))
    first = _check_at_scale(by_len, w.haystacks)
    assert np.array_equal(first, rows(by_len.find_leftmost_longest_batch(w.haystacks)))
