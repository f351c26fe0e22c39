"""Test-only restatement of the case-folded stream feeds (acb_streams_new_folded and every feed of such a batch,
csrc/acb_device.cu) on the stream restatements of tests/emul_streams.py, tests/emul_stream_leftmost.py,
tests/emul_stream_words.py and tests/emul_leftmost_first.py.  It replaces StreamBatch._native and ReplaceStream._native
of ascii_case_insensitive batches (other batches go on to whatever served them before), and stands in for their table:
the folded automaton's flat view (of Automaton._fold_host's trie), whose key ids are the group representatives.

A folded feed is the feed of the same form with every scan reading the folded text (emul_fold.fold, letter by letter:
the scans of tests/emul.py are wrapped for the call), while the staging, the held letters, the word flags and the
rewrite see the text as given.  The find_all forms then add every alias of each record's key right after it, ascending
(emul_fold.expand), as the device does before its commit; their records are already in the reference order, so a group
stays together in ascending id.  An emulated feed never overflows.
"""
from __future__ import annotations

import contextlib

import numpy as np

import emul
import emul_fold
import emul_leftmost_first
import emul_stream_leftmost
import emul_stream_words
import emul_streams


def fold_bytes(buf, L: int) -> np.ndarray:
    """the bytes of whole letters of width L with every letter 0x41..0x5A made small"""
    a = np.frombuffer(np.asarray(buf, dtype=np.uint8).tobytes(), dtype=np.uint8 if L == 1 else "<u4")
    return emul_fold.fold(a).astype(a.dtype).view(np.uint8)


@contextlib.contextmanager
def folded_scans(L: int):
    """emul.emul_filter and emul.emul_dfa read a folded copy of their text for the duration"""
    real = emul.emul_filter, emul.emul_dfa

    def wrap(scan):
        return lambda f, buf, *a, **k: scan(f, fold_bytes(buf, L), *a, **k)
    emul.emul_filter, emul.emul_dfa = wrap(real[0]), wrap(real[1])
    try:
        yield
    finally:
        emul.emul_filter, emul.emul_dfa = real


def expand(recs, core):
    """records [(chunk, end, key)] with every alias of their key after them (emul_fold.expand on the alias lists)"""
    if core is None or not len(core.alias_ids) or not recs:
        return recs
    out, _ = emul_fold.expand(np.array(recs, dtype=np.int64), core.alias_ptr.astype(np.int64), core.alias_ids.astype(np.int64),
                              1 << 60)
    return [tuple(r) for r in out.tolist()]


def _flat(A):
    """the table of a folded batch: the folded automaton, or the full one when there is no key"""
    core = A._fold_host(False)
    return A.flat() if core is None else A._flat_view(core.trie)


def _records(recs):
    from pyahocorasick_b200 import _native as N
    out = np.empty(len(recs), dtype=N.MATCH_DTYPE)
    for i, r in enumerate(recs):
        out[i] = r
    return out


def _state(self, words, leftmost):
    """what the device keeps per stream; L and T are those of the full automaton, as folding keeps every key's length"""
    A = self._A
    if words is not None:
        return emul_stream_words.new_state(A, self.n_streams, leftmost, words)
    st = emul_stream_leftmost._state(A, self.n_streams)
    if not leftmost:                                          # a find_all batch: the tail of emul_streams
        st.update(tail=[b""] * self.n_streams, state=[0] * self.n_streams)
    return st


def _common(self, op, args):
    st = self._ss
    if "bits" in st:
        return emul_stream_words._common(self, op, args)
    done, res = emul_stream_leftmost._common(self, st, op, args)
    if done and op == "reset" and "tail" in st:
        ids, = args
        for s in (range(self.n_streams) if ids is None else ids.tolist()):
            st["tail"][s] = b""
    return done, res


def install(monkeypatch, algo="filter"):
    """Route StreamBatch._native and ReplaceStream._native of ascii_case_insensitive batches through the emulation."""
    from pyahocorasick_b200 import _native as N
    from pyahocorasick_b200 import automaton as am

    real_stream, real_replace = am.StreamBatch._native, am.ReplaceStream._native

    def fake_stream(self, op, *args):
        if not self.ascii_case_insensitive:
            return real_stream(self, op, *args)
        leftmost = self.leftmost_longest or self.leftmost_first
        if op in ("new", "new_leftmost", "new_words"):
            return _state(self, self._words, leftmost)
        done, res = _common(self, op, args)
        if done:
            return res
        A = self._A
        f, core = _flat(A), A._fold_host(False)
        kind, data, offs, n, stride, ids, flag = args
        assert kind == "host"
        chunks = emul_stream_leftmost._chunks(data, offs, n, stride)
        a = algo if self._algo == "auto" else self._algo
        with folded_scans(f["letter_bytes"]):
            if op == "feed":
                return _records(expand(emul_streams.feed(f, self._ss, chunks, ids, a, False), core))
            if op == "feed_words":
                return _records(expand(emul_stream_words.feed(f, self._ss, chunks, ids, a, flag), core))
            if self.leftmost_first:
                return _records(emul_leftmost_first.feed(f, self._ss, chunks, ids, a, flag))
            if self.whole_words:
                return _records(emul_stream_words.feed(f, self._ss, chunks, ids, a, flag))
            return _records(emul_stream_leftmost.feed(f, self._ss, chunks, ids, a, flag))

    def fake_replace(self, op, *args):
        if not self.ascii_case_insensitive:
            return real_replace(self, op, *args)
        if op == "new":
            return _state(self, self._words, True)
        done, res = _common(self, op, args)
        if done:
            return res
        f = _flat(self._A)
        kind, data, offs, n, stride, ids, final = args
        assert kind == "host"
        rep, rep_off = self._R._tables[False]
        chunks = emul_stream_leftmost._chunks(data, offs, n, stride)
        a = algo if self._algo == "auto" else self._algo
        with folded_scans(f["letter_bytes"]):
            if self._R._select == N.SELECT_FIRST:
                return emul_leftmost_first.replace_feed(f, self._ss, chunks, ids, a, final, rep, rep_off)
            mod = emul_stream_words if self.whole_words else emul_stream_leftmost
            return mod.replace_feed(f, self._ss, chunks, ids, a, final, rep, rep_off)

    monkeypatch.setattr(am.StreamBatch, "_native", fake_stream)
    monkeypatch.setattr(am.ReplaceStream, "_native", fake_replace)
