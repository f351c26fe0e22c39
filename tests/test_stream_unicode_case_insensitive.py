"""Automaton.case_insensitive_stream_batch and Replacer.case_insensitive_stream_batch: over all feeds and `finish` of a
stream, what the whole-batch method gives with case_insensitive=True for the stream's whole text, whatever the chunk
cuts; and the C feeds refuse a table of the other fold (ASCII against Unicode and back)."""
import ctypes

import numpy as np
import pytest

import pyahocorasick_b200 as pkg
from batch_cases import triples
from pyahocorasick_b200 import _native as N
from pyahocorasick_b200.automaton import _FOLD_ASCII, _FOLD_UNICODE

ALPHABET = "kK\u212AsS\u017F\u00B5\u039C\u03BC\u03A3\u03C3\u03C2\u00C9\u00E9\u0178\u00FF\u00DF\u1E9E\u01C4\u01C5\u01C6" \
           "\U00010400\U00010428 a"


@pytest.fixture
def cta_limit():
    """limit(A, n): the CTA limit of A's Unicode-folded device-0 table of 4-byte letters (the one streams run on); set
    back to 0 after (A is kept alive until then: its tables go with it)"""
    seen = []

    def limit(A, n):
        tb = A._table_for(0, False, _FOLD_UNICODE)
        N.check(N.lib().acb_table_set_cta_limit(tb, n))
        seen.append((A, tb))
    yield limit
    for _, tb in seen:
        N.check(N.lib().acb_table_set_cta_limit(tb, 0))


def random_keys(rng):
    keys = []
    while len(keys) < int(rng.integers(2, 9)):
        k = "".join(rng.choice(list(ALPHABET), size=int(rng.integers(1, 5))))
        if k not in keys:
            keys.append(k)
        if rng.integers(0, 3) == 0 and k.swapcase() not in keys and len(k.swapcase()) == len(k):
            keys.append(k.swapcase())
    return keys


def cuts(rng, t, n_pieces):
    at = sorted(int(x) for x in rng.integers(0, len(t) + 1, size=n_pieces - 1))
    return [t[a:b] for a, b in zip([0] + at, at + [len(t)])]


def fed(make, texts, pieces, device=False):
    """the records of a StreamBatch over all feeds (and finish, where it has one), as sorted (stream, end, key) triples;
    device: equal-length chunks as CUDA tensors of 4-byte letters"""
    import torch
    S = make()
    out = []
    for r in range(max(len(p) for p in pieces)):
        chunk = [p[r] if r < len(p) else "" for p in pieces]
        if device:
            chunk = torch.from_numpy(np.array([[ord(c) for c in x] for x in chunk], dtype="<u4").view(np.uint8).copy()).cuda()
        out += triples(S.feed(chunk))
    if S.leftmost_longest or S.leftmost_first or S.whole_words:
        out += triples(S.finish())
    assert S.case_insensitive and not S.ascii_case_insensitive
    return sorted(out)


@pytest.mark.gpu
@pytest.mark.parametrize("limit", [0, 1])
def test_gpu_every_form_against_the_whole_batch(limit, cta_limit):
    rng = np.random.default_rng(41 + limit)
    for trial in range(6):
        keys = random_keys(rng)
        A = pkg.flavour("unicode").Automaton(pkg.flavour("unicode").STORE_INTS)
        for i, k in enumerate(keys):
            A.add_word(k, i)
        A.make_automaton()
        cta_limit(A, limit)
        texts = ["".join(rng.choice(list(ALPHABET), size=int(rng.integers(0, 60)))) for _ in range(5)]
        pieces = [cuts(rng, t, int(rng.integers(1, 7))) for t in texts]
        algo = ("filter", "dfa")[trial % 2]
        for ww in (False, True):
            whole = {"find_all": A.find_all_batch(texts, whole_words=ww, case_insensitive=True, algo=algo),
                     "longest": A.find_leftmost_longest_batch(texts, whole_words=ww, case_insensitive=True, algo=algo),
                     "first": A.find_leftmost_first_batch(texts, whole_words=ww, case_insensitive=True, algo=algo)}
            opts = {"find_all": {}, "longest": {"leftmost_longest": True}, "first": {"leftmost_first": True}}
            for form, o in opts.items():
                got = fed(lambda: A.case_insensitive_stream_batch(len(texts), algo=algo, whole_words=ww, **o), texts, pieces)
                assert got == sorted(triples(whole[form])), (keys, texts, pieces, form, ww)
            for first in (False, True):
                R = A.replacer({k: "<%d>" % i for i, k in enumerate(keys)}, leftmost_first=first)
                S = R.case_insensitive_stream_batch(len(texts), algo=algo, whole_words=ww)
                assert S.case_insensitive and not S.ascii_case_insensitive
                outs = ["" for _ in texts]
                for r in range(max(len(p) for p in pieces)):
                    for s, x in enumerate(S.feed([p[r] if r < len(p) else "" for p in pieces])):
                        outs[s] += x
                for s, x in enumerate(S.finish()):
                    outs[s] += x
                assert outs == R.replace_batch(texts, whole_words=ww, case_insensitive=True, algo=algo), (keys, texts, first)
        # CUDA tensor chunks of equal length
        texts = ["".join(rng.choice(list(ALPHABET), size=24)) for _ in range(4)]
        pieces = [[t[i:i + 6] for i in range(0, 24, 6)] for t in texts]
        for o, m in (({}, A.find_all_batch), ({"leftmost_longest": True}, A.find_leftmost_longest_batch)):
            got = fed(lambda: A.case_insensitive_stream_batch(len(texts), **o), texts, pieces, device=True)
            assert got == sorted(triples(m(texts, case_insensitive=True)))


@pytest.mark.gpu
def test_gpu_c_feeds_refuse_the_other_fold():
    A = pkg.flavour("unicode").Automaton()
    for i, k in enumerate(["ab", "AB", "é"]):
        A.add_word(k, i)
    A.make_automaton()
    L = N.lib()
    asc, uni = A._table_for(0, False, _FOLD_ASCII), A._table_for(0, False, _FOLD_UNICODE)
    flat = np.frombuffer("abcd".encode("utf-32-le"), dtype=np.uint8).copy()
    out = np.zeros(8 * 3, dtype=np.int32)
    found = ctypes.c_int64()
    for made, other in ((asc, uni), (uni, asc)):
        for leftmost in (0, 1):
            ss = ctypes.c_void_p()
            N.check(L.acb_streams_new_folded(made, 2, leftmost, N.SELECT_LONGEST, None, -1, ctypes.byref(ss)))
            try:
                if leftmost:
                    feed = lambda tb: L.acb_streams_feed_leftmost_host(ss, tb, N.ptr(flat), 16, None, 1, 16, None, 0, N.ptr(out), 8,
                                                                       ctypes.byref(found), 0)
                else:
                    feed = lambda tb: L.acb_streams_feed_host(ss, tb, N.ptr(flat), 16, None, 1, 16, None, N.ptr(out), 8,
                                                              ctypes.byref(found), 0, 1)
                assert feed(other) == N.ACB_EINVAL
                assert "its own fold" in N.last_error()
                assert feed(made) == N.ACB_OK
            finally:
                L.acb_streams_free(ss)
    S = A.case_insensitive_stream_batch(1)
    T = A.ascii_case_insensitive_stream_batch(1)
    assert triples(S.feed(["xAbÉ"])) == [(0, 2, 0), (0, 2, 1), (0, 3, 2)]
    assert triples(T.feed(["xAbÉ"])) == [(0, 2, 0), (0, 2, 1)]
    assert not T.case_insensitive and T.ascii_case_insensitive
    assert not A.stream_batch(1).case_insensitive and not A.stream_batch(1).ascii_case_insensitive
