"""Test-only restatement of the whole-word stream feeds (acb_streams_new_words; acb_streams_feed_words_*,
acb_streams_feed_leftmost_* and acb_streams_replace_* on such a batch, csrc/acb_device.cu) in Python, on the staging of
tests/emul_stream_leftmost.py, the scans of tests/emul.py, the word flags of tests/emul_words.py, the selection of
tests/emul_leftmost.py and the replacement passes of tests/emul_replace.py.  It replaces StreamBatch._native and
ReplaceStream._native for whole-word batches (other batches go on to whatever served them before), so that the CPU suite
runs the Python layer against it.

Per stream it keeps what the device keeps: the position, up to T + 1 held letters and `left`, whether the letter just
before the held ones is a word letter.  A feed stages held || chunk per chunk, scans the staged batch and keeps the
whole-word records of its window -- a record that starts at staged letter 0 takes its left neighbour from `left`:
  - leftmost: records that start before staged_len - T - 1 (all on a final feed), then the selection, and the new X
    max(0, staged_len - T - 1, last chosen end + 1);
  - find_all: records that end in [held - 1, staged_len - 2] (staged_len - 1 on a final feed), ordered by chunk, end,
    longest key first, and the new X max(0, staged_len - T - 1).
A final feed moves X to staged_len.  The commit keeps the letters after X, and sets `left` from staged letter X - 1
(unchanged when X is 0; cleared by a final feed).  An emulated feed never overflows.
"""
from __future__ import annotations

import numpy as np

import emul
import emul_leftmost
import emul_replace
import emul_stream_leftmost
import emul_words


def _word(st, v: int) -> bool:
    return v < st["n_bits"] and bool(int(st["bits"][v >> 5]) >> (v & 31) & 1)


def _letter(flat, at: int, L: int) -> int:
    return int.from_bytes(flat[at:at + L].tobytes(), "little")


def settle(f, st, flat, offs, held, ids, algo, final):
    """scan, window, word flags, then selection (leftmost) or order (find_all) -> (records (n, 3) in staged coordinates,
    new X per chunk in staged letters)"""
    L, H = st["L"], st["T"] + 1
    kl = np.asarray(f["key_len"], dtype=np.int64)
    n = len(offs) - 1
    scan = emul.emul_dfa if algo == "dfa" else emul.emul_filter
    full = np.array(scan(f, flat, offs) if flat.size else [], dtype=np.int64).reshape(-1, 3)
    staged_len = np.diff(offs) // L
    h, e = full[:, 0], full[:, 1]
    start = e - kl[full[:, 2]] + 1
    hl = np.asarray(held, dtype=np.int64)
    if st["leftmost"]:
        window = np.ones(len(full), dtype=bool) if final else start < staged_len[h] - H
    else:
        window = (e >= hl[h] - 1) & (e <= staged_len[h] - 2 + int(final))
    assert final or (e[window] + 1 < staged_len[h[window]]).all()      # the right neighbour is staged
    sid = np.arange(n) if ids is None else np.asarray(ids, dtype=np.int64)
    left = np.array([st["left"][s] for s in sid], dtype=bool)
    whole = emul_words.flags(flat, offs, 0, L, full, kl, st["bits"], st["n_bits"]) & ~((start == 0) & left[h])
    kept = full[window & whole]
    if st["leftmost"]:
        kept = emul_leftmost.select(kept, kl, int(kl.max()) if len(kl) else 0)
    else:
        kept = kept[np.lexsort((-kl[kept[:, 2]], kept[:, 1], kept[:, 0]))]
    last = np.full(n, -1, dtype=np.int64)
    if st["leftmost"]:
        for c, end, _ in kept.tolist():
            last[c] = end
    xn = staged_len.copy() if final else np.maximum(np.maximum(staged_len - H, 0), last + 1)
    return kept, xn


def commit(st, chunks, ids, flat, offs, xn, final):
    L = st["L"]
    for h in range(len(chunks)):
        s = h if ids is None else int(ids[h])
        if final:
            st["left"][s] = False
        elif xn[h] > 0:
            st["left"][s] = _word(st, _letter(flat, int(offs[h] + (xn[h] - 1) * L), L))
    emul_stream_leftmost.commit(st, chunks, ids, flat, offs, xn, final)


def feed(f, st, chunks, ids, algo, final):
    """a find_all or leftmost word feed -> its records [(chunk, end relative to the chunk, key)]"""
    flat, offs, held = emul_stream_leftmost.stage(st, chunks, ids)
    kept, xn = settle(f, st, flat, offs, held, ids, algo, final)
    commit(st, chunks, ids, flat, offs, xn, final)
    return [(h, e - held[h], k) for h, e, k in kept.tolist()]


def replace_feed(f, st, chunks, ids, algo, final, rep, rep_off, tile=4096):
    """the replacing word feed -> (output bytes, output offsets)"""
    L = st["L"]
    flat, offs, held = emul_stream_leftmost.stage(st, chunks, ids)
    chosen, xn = settle(f, st, flat, offs, held, ids, algo, final)
    win = np.concatenate([flat[offs[h]:offs[h] + xn[h] * L] for h in range(len(chunks))]) if chunks else np.empty(0, np.uint8)
    woff = np.zeros(len(chunks) + 1, dtype=np.int64)
    np.cumsum(xn * L, out=woff[1:])
    out, out_off = emul_replace.replace(win, woff, chosen, f["key_len"], rep, rep_off, L, tile)
    commit(st, chunks, ids, flat, offs, xn, final)
    return out, out_off


def new_state(A, n_streams, leftmost, words):
    from pyahocorasick_b200.automaton import _word_bits
    f = A.flat()
    L = f["letter_bytes"]
    bits, n_bits = _word_bits(words, L)
    return {"L": L, "T": max(f["max_key_bytes"] // L - 1, 0), "pos": np.zeros(n_streams, dtype=np.int64),
            "held": [b""] * n_streams, "left": [False] * n_streams, "leftmost": leftmost, "bits": bits, "n_bits": n_bits}


def _common(self, op, args):
    done, res = emul_stream_leftmost._common(self, self._ss, op, args)
    if done and op == "reset":
        ids, = args
        for s in (range(self.n_streams) if ids is None else ids.tolist()):
            self._ss["left"][s] = False
    return done, res


def install(monkeypatch, algo="filter", tile=4096):
    """Route StreamBatch._native and ReplaceStream._native of whole-word batches through the emulation."""
    from pyahocorasick_b200 import _native as N
    from pyahocorasick_b200 import automaton as am

    real_stream, real_replace = am.StreamBatch._native, am.ReplaceStream._native

    def fake_stream(self, op, *args):
        if not self.whole_words:
            return real_stream(self, op, *args)
        if op == "new_words":
            return new_state(self._A, self.n_streams, self.leftmost_longest, self._words)
        done, res = _common(self, op, args)
        if done:
            return res
        assert op == ("feed_leftmost" if self.leftmost_longest else "feed_words")
        kind, data, offs, n, stride, ids, final = args
        assert kind == "host"
        recs = feed(self._A.flat(), self._ss, emul_stream_leftmost._chunks(data, offs, n, stride), ids,
                    algo if self._algo == "auto" else self._algo, final)
        out = np.empty(len(recs), dtype=N.MATCH_DTYPE)
        for i, r in enumerate(recs):
            out[i] = r
        return out

    def fake_replace(self, op, *args):
        if not self.whole_words:
            return real_replace(self, op, *args)
        if op == "new":
            return new_state(self._A, self.n_streams, True, self._words)
        done, res = _common(self, op, args)
        if done:
            return res
        kind, data, offs, n, stride, ids, final = args
        assert kind == "host"
        rep, rep_off = self._R._tables[False]
        return replace_feed(self._A.flat(), self._ss, emul_stream_leftmost._chunks(data, offs, n, stride), ids,
                            algo if self._algo == "auto" else self._algo, final, rep, rep_off, tile)

    monkeypatch.setattr(am.StreamBatch, "_native", fake_stream)
    monkeypatch.setattr(am.ReplaceStream, "_native", fake_replace)
