"""Every batch route of the Python layer, once on a host batch and once on a CUDA tensor, from a fresh automaton whose
first guess of the record (or output) room is too small: the route must retry once with the exact size, return what
the same call returns with room to spare, and make exactly the native calls pinned below.

The calls are recorded by a forwarding proxy in place of the automaton's library.  The acb_trie_* queries and
acb_release_records are left out: the latter runs when the garbage collector frees a record buffer, at no fixed time.
Each haystack is a few thousand whole words, so one call has more records than the first guess
max(match_cap, 4096, 2 * n) and a replacement more output bytes than size * 5 // 4 + 4096."""
import numpy as np
import pytest

import pyahocorasick_b200 as pkg
from pyahocorasick_b200 import automaton as am

REPLACEMENTS = {"a": "<A>", "b": "<B>", "ab": "<AB-REPLACED>"}
N_HAY, REPS = 2, 3000                              # 2 * 3000 "ab" per call: more than 4096 records on every route
FIRST_GUESS = 1 << 12

UP = "acb_table_upload"
SCAN, SCAN_DEV, SORT_DEV, TAKE = "acb_scan_host", "acb_scan_device", "acb_sort_matches_device", "acb_take_records"
WORDS_DEV, SELECT_DEV = "acb_word_filter_device", "acb_leftmost_longest_device"
REPLACER = "acb_replacer_new"

CALLS = {
    # upload the table; scan, overflow, scan again, take records
    ("find_all", "host"): [UP, SCAN, SCAN, TAKE],
    # upload the table; scan, count past the room, scan again, sort on the device
    ("find_all", "device"): [UP, SCAN_DEV, SCAN_DEV, SORT_DEV],
    ("white_space", "host"): [UP, "acb_scan_host_skip", "acb_scan_host_skip", TAKE],
    ("white_space", "device"): [UP, "acb_scan_device_skip", "acb_scan_device_skip", SORT_DEV],
    ("whole_words", "host"): [UP, "acb_scan_host_words", "acb_scan_host_words", TAKE],
    # ... scan, scan again, keep the whole words, sort
    ("whole_words", "device"): [UP, SCAN_DEV, SCAN_DEV, WORDS_DEV, SORT_DEV],
    ("long", "host"): [UP, SCAN, SCAN, TAKE],
    ("long", "device"): [UP, SCAN_DEV, SCAN_DEV, SORT_DEV],
    # upload the latin-1 table; scan, overflow, scan again, take records
    ("latin1", "host"): [UP, SCAN, SCAN, TAKE],
    ("latin1", "device"): [UP, SCAN_DEV, SCAN_DEV, SORT_DEV],
    ("leftmost", "host"): [UP, "acb_scan_host_leftmost", "acb_scan_host_leftmost", TAKE],
    # ... full scan, full scan again, select
    ("leftmost", "device"): [UP, SCAN_DEV, SCAN_DEV, SELECT_DEV],
    ("leftmost_words", "host"): [UP, "acb_scan_host_leftmost_words", "acb_scan_host_leftmost_words", TAKE],
    ("leftmost_words", "device"): [UP, SCAN_DEV, SCAN_DEV, WORDS_DEV, SELECT_DEV],
    # upload the table and the replacements; rewrite, overflow, rewrite again
    ("replace", "host"): [UP, REPLACER, "acb_replace_host", "acb_replace_host"],
    # ... select as above, upload the replacements, count the output, write it
    ("replace", "device"): [UP, SCAN_DEV, SCAN_DEV, SELECT_DEV, REPLACER, "acb_replace_device", "acb_replace_device"],
    ("replace_words", "host"): [UP, REPLACER, "acb_replace_host_words", "acb_replace_host_words"],
    ("replace_words", "device"): [UP, SCAN_DEV, SCAN_DEV, WORDS_DEV, SELECT_DEV, REPLACER, "acb_replace_device",
                                  "acb_replace_device"],
    # stream batches (table made with the batch): feed, overflow, feed again, take records
    ("feed", "host"): ["acb_streams_feed_host", "acb_streams_feed_host", TAKE],
    # feed, count past the room, feed again, sort on the device
    ("feed", "device"): ["acb_streams_feed_device", "acb_streams_feed_device", SORT_DEV],
    ("feed_white_space", "host"): ["acb_streams_feed_host", "acb_streams_feed_host", TAKE],
    ("feed_white_space", "device"): ["acb_streams_feed_device", "acb_streams_feed_device", SORT_DEV],
    ("feed_long", "host"): ["acb_streams_feed_host", "acb_streams_feed_host", TAKE],
    ("feed_long", "device"): ["acb_streams_feed_device", "acb_streams_feed_device", SORT_DEV],
    # feed, overflow, feed again, take records; finish: one final feed that settles nothing more
    ("feed_leftmost", "host"): ["acb_streams_feed_leftmost_host", "acb_streams_feed_leftmost_host", TAKE,
                                "acb_streams_feed_leftmost_host"],
    ("feed_leftmost", "device"): ["acb_streams_feed_leftmost_device", "acb_streams_feed_leftmost_device",
                                  "acb_streams_feed_leftmost_host"],
    # upload the replacements; rewrite, overflow, rewrite again; finish: one final rewrite
    ("replace_stream", "host"): [REPLACER, "acb_streams_replace_host", "acb_streams_replace_host",
                                 "acb_streams_replace_host"],
    ("replace_stream", "device"): [REPLACER, "acb_streams_replace_device", "acb_streams_replace_device",
                                   "acb_streams_replace_host"],
    # per chunk: set the state, scan, overflow, set it again, scan again, read the end state, take records
    ("iter_long", "host"): [UP] + 2 * ["acb_table_set_long_state", SCAN, "acb_table_set_long_state", SCAN,
                                       "acb_table_get_long_state", TAKE],
}

RECORD_ROUTES = {"find_all", "white_space", "whole_words", "long", "latin1", "leftmost", "leftmost_words", "feed",
                 "feed_white_space", "feed_long", "feed_leftmost", "iter_long"}


class _Recorder:
    """Forwards every attribute to the library and records the name of each acb_* function called"""

    def __init__(self, lib):
        self._lib = lib
        self.calls = []

    def __getattr__(self, name):
        fn = getattr(self._lib, name)
        if not name.startswith("acb_") or name.startswith("acb_trie_") or name == "acb_release_records":
            return fn

        def call(*args):
            self.calls.append(name)
            return fn(*args)
        return call


def _automaton(unicode=False):
    m = pkg.flavour("unicode" if unicode else "bytes")
    A = m.Automaton(m.STORE_ANY)
    for k, v in REPLACEMENTS.items():
        if unicode:
            A.add_word(k, v)
        else:
            A.add_word(k.encode(), v.encode())
    A.make_automaton()
    return A


def _hays(unicode=False, reps=REPS):
    h = "ab " * reps
    return [h] * N_HAY if unicode else [h.encode()] * N_HAY


def _form(hays, form):
    """the batch in one of find_all_batch's input forms"""
    import torch
    raw = [h.encode("utf-32-le") if isinstance(h, str) else h for h in hays]
    if form == "list":
        return list(hays)
    if form == "array":
        return np.frombuffer(b"".join(raw), dtype=np.uint8).reshape(len(raw), -1).copy()
    if form == "pair":
        return np.frombuffer(b"".join(raw), dtype=np.uint8).copy(), np.cumsum([0] + [len(r) for r in raw]).astype(np.int64)
    return torch.frombuffer(bytearray(b"".join(raw)), dtype=torch.uint8).reshape(len(raw), -1).cuda()


def _plain(r):
    """a result as nested lists, to compare"""
    if isinstance(r, am.Matches):
        return r.hay_id.tolist(), r.end_index.tolist(), r.key_id.tolist()
    if isinstance(r, (tuple, list)) and r and not isinstance(r[0], (str, bytes)):
        return [_plain(x) for x in r]
    if hasattr(r, "cpu"):
        return r.cpu().numpy().tolist()
    if isinstance(r, np.ndarray):
        return r.tolist()
    return r


def _run(route, A, batch):
    """the route's call (or feeds) on A -> result; streams and replacers are made before the calls are recorded"""
    if route in ("find_all", "latin1"):
        return lambda: A.find_all_batch(batch)
    if route == "white_space":
        return lambda: A.find_all_batch(batch, ignore_white_space=True)
    if route == "whole_words":
        return lambda: A.find_all_batch(batch, whole_words=True)
    if route == "long":
        return lambda: A.find_all_batch(batch, algo="long")
    if route == "leftmost":
        return lambda: A.find_leftmost_longest_batch(batch)
    if route == "leftmost_words":
        return lambda: A.find_leftmost_longest_batch(batch, whole_words=True)
    if route in ("replace", "replace_words"):
        R = A.replacer()
        return lambda: R.replace_batch(batch, whole_words=route == "replace_words")
    if route == "replace_stream":
        S = A.replacer().stream_batch(N_HAY)
        return lambda: (S.feed(batch), S.finish())
    S = A.stream_batch(N_HAY, long=route == "feed_long", ignore_white_space=route == "feed_white_space",
                       leftmost_longest=route == "feed_leftmost")
    if route == "feed_leftmost":
        return lambda: (S.feed(batch), S.finish())
    return lambda: S.feed(batch)


CASES = [(r, f) for r in ("find_all", "white_space", "whole_words", "long", "leftmost", "leftmost_words", "replace",
                          "replace_words", "feed", "feed_white_space", "feed_long", "feed_leftmost", "replace_stream")
         for f in ("list", "array", "pair", "cuda")] + [("latin1", "list"), ("latin1", "cuda")]


@pytest.mark.gpu
@pytest.mark.parametrize("route,form", CASES)
def test_batch_route_retries_once_with_the_exact_size(route, form):
    unicode = route == "latin1"
    ref = _automaton(unicode)
    ref._match_cap = 1 << 20
    want = _plain(_run(route, ref, _form(_hays(unicode), form))())

    A = _automaton(unicode)
    assert A._match_cap == 0
    rec = A._lib = _Recorder(A._lib)
    call = _run(route, A, _form(_hays(unicode), form))
    rec.calls = []
    got = call()
    assert rec.calls == CALLS[(route, "device" if form == "cuda" else "host")]
    assert _plain(got) == want
    if route in RECORD_ROUTES:
        assert A._match_cap > FIRST_GUESS


def _iter_long(A, chunks):
    it = A.iter_long(chunks[0])
    out = [list(it)]
    it.set(chunks[1])
    out.append(list(it))
    return out


@pytest.mark.gpu
def test_iter_long_retries_each_chunk_with_its_state():
    chunks = [("ab " * 5000).encode(), ("ab " * 8000).encode()]          # the second outgrows the room the first left
    ref = _automaton()
    ref._match_cap = 1 << 20
    want = _iter_long(ref, chunks)
    assert [len(w) for w in want] == [5000, 8000]

    A = _automaton()
    rec = A._lib = _Recorder(A._lib)
    assert _iter_long(A, chunks) == want
    assert rec.calls == CALLS[("iter_long", "host")]
    assert A._match_cap > 5000 + 1024
