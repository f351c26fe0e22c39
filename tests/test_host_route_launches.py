"""Kernel launches (acb_launch_count) of every host-buffer entry point on one small fixed batch.

The host routes share their upload, read-back, timing and launch-check code; the counts pin what each route launches,
so that sharing cannot add, drop or regroup a launch.  Each constant names the launches it counts.  cub calls are not
counted.  The batch is small (one scan segment, no pipelined scan), has more than one match per route (so the record sort
runs), and every leftmost feed is final (every match is settled and chosen in the same feed).
"""
import ctypes

import numpy as np
import pytest

from pyahocorasick_b200 import _native as N
from pyahocorasick_b200 import synth
from pyahocorasick_b200.automaton import _word_bits

KEYS = [b"he", b"she", b"his", b"hers"]
HAYS = [b"ushers and she sells his shells", b"his hers", b"", b"hehe she said"]
CAP = 1024
AT_LEAST_PREFIX = 2                                           # ACB_MATCH_AT_LEAST_PREFIX
WORD_BITS, N_WORD_BITS = _word_bits(("bytes", None), 1)        # the default word set of the acb_*_words routes


def _batch():
    flat = np.frombuffer(b"".join(HAYS), dtype=np.uint8).copy()
    off = np.cumsum([0] + [len(h) for h in HAYS]).astype(np.int64)
    return flat, off


def _records(L, call):
    """call(out, n_found) on a fresh record buffer; the record count, checked to be > 1"""
    out = np.empty((CAP, 3), dtype=np.int32)
    n = ctypes.c_int64()
    N.check(call(N.ptr(out), ctypes.byref(n)))
    assert n.value > 1
    return n.value


def _scan_host(L, A, tb, flat, off):
    _records(L, lambda out, n: L.acb_scan_host(tb, N.ptr(flat), flat.size, N.ptr(off), len(off) - 1, 0, out, CAP, n,
                                               N.ALGO_FILTER, 1))


def _scan_host_skip(L, A, tb, flat, off):
    skip = np.array([ord(" ")], dtype=np.uint32)
    _records(L, lambda out, n: L.acb_scan_host_skip(tb, N.ptr(flat), flat.size, N.ptr(off), len(off) - 1, 0, out, CAP, n,
                                                    N.ALGO_FILTER, 1, N.ptr(skip), skip.size))


def _feed(L, tb, ss, flat, off, algo):
    _records(L, lambda out, n: L.acb_streams_feed_host(ss, tb, N.ptr(flat), flat.size, N.ptr(off), len(off) - 1, 0, None,
                                                       out, CAP, n, algo, 1))


def _with_streams(L, make, use):
    ss = ctypes.c_void_p()
    N.check(make(ctypes.byref(ss)))
    try:
        use(ss)
    finally:
        L.acb_streams_free(ss)


def _feed_find_all(L, A, tb, flat, off):
    _with_streams(L, lambda p: L.acb_streams_new(tb, len(HAYS), 0, p), lambda ss: _feed(L, tb, ss, flat, off, N.ALGO_FILTER))


def _feed_skip(L, A, tb, flat, off):
    skip = np.array([ord(" ")], dtype=np.uint32)
    _with_streams(L, lambda p: L.acb_streams_new_skip(tb, len(HAYS), N.ptr(skip), skip.size, p),
                  lambda ss: _feed(L, tb, ss, flat, off, N.ALGO_FILTER))


def _feed_long(L, A, tb, flat, off):
    _with_streams(L, lambda p: L.acb_streams_new(tb, len(HAYS), 1, p), lambda ss: _feed(L, tb, ss, flat, off, N.ALGO_LONG))


def _lookup_host(L, A, tb, flat, off):
    key_id = np.empty(len(HAYS), dtype=np.int32)
    prefix = np.empty(len(HAYS), dtype=np.int32)
    N.check(L.acb_lookup_host(tb, N.ptr(flat), flat.size, N.ptr(off), len(off) - 1, 0, N.ptr(key_id), N.ptr(prefix)))


def _select_host(L, A, tb, flat, off):
    pat = np.frombuffer(b"hs", dtype=np.uint8).copy()
    pat_off = np.array([0, 1, 2], dtype=np.int64)
    out_off = np.empty(3, dtype=np.int64)
    key_id = np.empty(CAP, dtype=np.int32)
    total = ctypes.c_int64()
    N.check(L.acb_select_host(tb, N.ptr(pat), pat.size, N.ptr(pat_off), 2, 0, -1, AT_LEAST_PREFIX, N.ptr(out_off),
                              N.ptr(key_id), CAP, ctypes.byref(total)))
    assert total.value == len(KEYS)


def _scan_host_leftmost(L, A, tb, flat, off):
    _records(L, lambda out, n: L.acb_scan_host_leftmost(tb, N.ptr(flat), flat.size, N.ptr(off), len(off) - 1, 0, out, CAP, n,
                                                        N.ALGO_FILTER))


def _with_replacer(L, tb, use):
    rep = np.frombuffer(b"".join(k.upper() + b"!" for k in KEYS), dtype=np.uint8).copy()
    rep_off = np.cumsum([0] + [len(k) + 1 for k in KEYS]).astype(np.int64)
    r = ctypes.c_void_p()
    N.check(L.acb_replacer_new(tb, N.ptr(rep), rep.size, N.ptr(rep_off), len(KEYS), ctypes.byref(r)))
    try:
        out_off = np.empty(len(HAYS) + 1, dtype=np.int64)
        out = np.empty(4096, dtype=np.uint8)
        total = ctypes.c_int64()
        N.check(use(r, N.ptr(out_off), N.ptr(out), out.size, ctypes.byref(total)))
        assert total.value > 0
    finally:
        L.acb_replacer_free(r)


def _replace_host(L, A, tb, flat, off):
    _with_replacer(L, tb, lambda r, oo, o, oc, t: L.acb_replace_host(r, tb, N.ptr(flat), flat.size, N.ptr(off), len(off) - 1, 0,
                                                                     N.ALGO_FILTER, oo, o, oc, t))


def _word_batch(tb, flat, off):
    return tb, N.ptr(flat), flat.size, N.ptr(off), len(off) - 1, 0, N.ptr(WORD_BITS), N_WORD_BITS


def _scan_host_words(L, A, tb, flat, off):
    _records(L, lambda out, n: L.acb_scan_host_words(*_word_batch(tb, flat, off), out, CAP, n, N.ALGO_FILTER, 1))


def _scan_host_leftmost_words(L, A, tb, flat, off):
    _records(L, lambda out, n: L.acb_scan_host_leftmost_words(*_word_batch(tb, flat, off), out, CAP, n, N.ALGO_FILTER))


def _replace_host_words(L, A, tb, flat, off):
    _with_replacer(L, tb, lambda r, oo, o, oc, t: L.acb_replace_host_words(r, *_word_batch(tb, flat, off), N.ALGO_FILTER, oo, o,
                                                                           oc, t))


def _feed_leftmost(L, A, tb, flat, off):
    _with_streams(L, lambda p: L.acb_streams_new_leftmost(tb, len(HAYS), p),
                  lambda ss: _records(L, lambda out, n: L.acb_streams_feed_leftmost_host(
                      ss, tb, N.ptr(flat), flat.size, N.ptr(off), len(off) - 1, 0, None, 1, out, CAP, n, N.ALGO_FILTER)))


def _streams_replace(L, A, tb, flat, off):
    _with_streams(L, lambda p: L.acb_streams_new_leftmost(tb, len(HAYS), p),
                  lambda ss: _with_replacer(L, tb, lambda r, oo, o, oc, t: L.acb_streams_replace_host(
                      ss, r, tb, N.ptr(flat), flat.size, N.ptr(off), len(off) - 1, 0, None, 1, N.ALGO_FILTER, oo, o, oc, t)))


# the leftmost-longest selection (acb_leftmost_longest_device, one sort pass): sort key, candidates, successors, chain,
# emit + count
SELECTION = 1 + 1 + 1 + 1 + 2
# the replacement (rp_offsets, rp_write): delta, records, offsets, tiles, write
REPLACEMENT = 3 + 2
# the whole-word filter (acb_word_filter_device): flags, emit + count
WORD_FILTER = 1 + 2
# a final leftmost feed up to its selection: staged lengths, gather tiles + gather, scan, frontier flags, then last chosen
# and frontier after it
FEED_LEFTMOST = 1 + 2 + 1 + 1 + 1 + 1

CASES = {
    "scan_host": (_scan_host, 1 + 1),                          # monolithic: stream/pair kernel, sort key
    "scan_host_skip": (_scan_host_skip, 2 + 1 + 1 + 1),        # compaction + offsets, scan, remap, sort key
    "feed_find_all": (_feed_find_all, 1 + 1 + 1 + 1),          # scan, seam, commit, sort key
    "feed_skip": (_feed_skip, 2 + 1 + 1 + 1 + 1 + 1),          # compaction + offsets, scan, seam, remap, commit, sort key
    "feed_long": (_feed_long, 2 + 1 + 1),                      # gather + iter_long, commit, sort key
    "lookup_host": (_lookup_host, 1),                          # lookup
    "select_host": (_select_host, 1 + 1),                      # count pass, fill pass
    "scan_host_leftmost": (_scan_host_leftmost, 1 + SELECTION),                # scan, selection
    "replace_host": (_replace_host, 1 + SELECTION + REPLACEMENT),              # scan, selection, replacement
    "feed_leftmost": (_feed_leftmost, FEED_LEFTMOST + SELECTION + 1),          # feed, selection, commit
    "streams_replace": (_streams_replace, FEED_LEFTMOST + SELECTION + 2 + REPLACEMENT + 1),   # ... window gather, replacement, commit
    "scan_host_words": (_scan_host_words, 1 + WORD_FILTER + 1),                                 # scan, word filter, sort key
    "scan_host_leftmost_words": (_scan_host_leftmost_words, 1 + WORD_FILTER + SELECTION),       # scan, word filter, selection
    "replace_host_words": (_replace_host_words, 1 + WORD_FILTER + SELECTION + REPLACEMENT),     # ... replacement
}


@pytest.mark.gpu
@pytest.mark.parametrize("route", sorted(CASES))
def test_host_route_launch_count(route):
    run, want = CASES[route]
    A = synth.build_automaton(KEYS)
    L = N.lib()
    tb = A._ensure_table(0)
    N.check(L.acb_table_upload_key_ranges(tb, A._trie))
    flat, off = _batch()
    run(L, A, tb, flat, off)                                  # first call: every workspace is grown
    before = L.acb_launch_count()
    run(L, A, tb, flat, off)
    assert L.acb_launch_count() - before == want
