"""Test-only restatement of the leftmost-first selection (acb_leftmost_first_device) and of the leftmost-first routes
built on it, for the CPU suite.  `greedy_first` is the definition the tests pin, stated directly.  `select_first` runs the
device's steps: re-key by hay | start | key_id and sort, then the leftmost-longest steps unchanged (the first record of
every (hay, start) run, its successor, the chain marking of tests/emul_leftmost.py, emit).  The stream feeds restate
acb_streams_feed_leftmost_* / acb_streams_replace_* on a leftmost-first batch with the staging and commit of
tests/emul_stream_leftmost.py and tests/emul_stream_words.py.  `install` routes the leftmost-first paths of the Python
layer through all of this on top of the emulated scan (tests/emul.py); leftmost-longest calls go on to whatever served
them before."""
from __future__ import annotations

import numpy as np

import emul
import emul_leftmost
import emul_replace
import emul_stream_leftmost
import emul_stream_words
import emul_words


def greedy_first(recs, key_len=None):
    """The definition over a full match list [(hay, end, key)]: per haystack, p = 0; take the smallest start >= p, the
    match there with the smallest key id, continue at its end + 1.  key_len[key] gives the start.  Returns the chosen
    records in haystack order, then end ascending."""
    by_hay = {}
    for h, e, k in recs:
        by_hay.setdefault(int(h), []).append((int(e) - int(key_len[k]) + 1, int(k), int(e)))
    out = []
    for h in sorted(by_hay):
        p = 0
        for s, k, e in sorted(by_hay[h]):
            if s >= p:
                out.append((h, e, k))
                p = e + 1
    return out


def select_first(rec, key_len, max_len: int, tile: int = 2048) -> np.ndarray:
    """acb_leftmost_first_device's steps on (n, 3) int records (hay, end, key) in any order -> the chosen records"""
    rec = np.asarray(rec, dtype=np.int64).reshape(-1, 3)
    key_len = np.asarray(key_len, dtype=np.int64)
    if len(rec) == 0:
        return np.empty((0, 3), dtype=np.int64)
    ln = key_len[rec[:, 2]]
    start = rec[:, 1] - ln + 1
    order = np.lexsort((rec[:, 2], start, rec[:, 0]))          # 1. hay | start | key_id, stable
    hay, start, ln, srt = rec[order, 0], start[order], ln[order], rec[order]
    first = np.ones(len(srt), dtype=bool)                      # 2. the first record of every (hay, start) run
    first[1:] = (hay[1:] != hay[:-1]) | (start[1:] != start[:-1])
    cand, chay, cstart, clen = srt[first], hay[first], start[first], ln[first]
    M = len(cand)
    nxt = np.full(M, -1, dtype=np.int64)                       # 3. successors, searched in [i + 1, i + len_i]
    for i in range(M):
        lo, hi = i + 1, min(M, i + int(clen[i]) + 1)
        target = cstart[i] + clen[i]
        while lo < hi:
            mid = (lo + hi) // 2
            if chay[mid] != chay[i] or cstart[mid] >= target:
                hi = mid
            else:
                lo = mid + 1
        if lo < M and chay[lo] == chay[i] and cstart[lo] >= target:
            nxt[i] = lo
    return cand[emul_leftmost.chain(chay, nxt, max(max_len, 1), tile)]   # 4. chain marking (asserts early exits), 5. emit


def _records(rows):
    from pyahocorasick_b200 import _native as N
    out = np.empty(len(rows), dtype=N.MATCH_DTYPE)
    for i, r in enumerate(np.asarray(rows, dtype=np.int64).reshape(-1, 3).tolist()):
        out[i] = tuple(r)
    return out


def _raw(full):
    if len(full) == 0:
        return np.empty((0, 3), dtype=np.int64)
    return np.stack([full["hay_id"], full["end_index"], full["key_id"]], axis=1).astype(np.int64)


# ------------------------------------------------------------------ stream feeds
def settle(f, st, flat, offs, held, ids, algo, final, tile):
    """scan, window (and word flags), leftmost-first selection -> (chosen (n, 3) staged coordinates, new X per chunk)"""
    L, H = st["L"], st["T"] + (1 if "bits" in st else 0)
    kl = np.asarray(f["key_len"], dtype=np.int64)
    n = len(offs) - 1
    scan = emul.emul_dfa if algo == "dfa" else emul.emul_filter
    full = np.array(scan(f, flat, offs) if flat.size else [], dtype=np.int64).reshape(-1, 3)
    staged_len = np.diff(offs) // L
    h = full[:, 0]
    start = full[:, 1] - kl[full[:, 2]] + 1
    keep = np.ones(len(full), dtype=bool) if final else start < staged_len[h] - H
    if "bits" in st:
        sid = np.arange(n) if ids is None else np.asarray(ids, dtype=np.int64)
        left = np.array([st["left"][s] for s in sid], dtype=bool)
        keep &= emul_words.flags(flat, offs, 0, L, full, kl, st["bits"], st["n_bits"]) & ~((start == 0) & left[h])
    chosen = select_first(full[keep], kl, int(kl.max()) if len(kl) else 0, tile)
    last = np.full(n, -1, dtype=np.int64)
    for c, e, _ in chosen.tolist():
        last[c] = e
    xn = staged_len.copy() if final else np.maximum(np.maximum(staged_len - H, 0), last + 1)
    return chosen, xn


def _commit(st, chunks, ids, flat, offs, xn, final):
    (emul_stream_words.commit if "bits" in st else emul_stream_leftmost.commit)(st, chunks, ids, flat, offs, xn, final)


def feed(f, st, chunks, ids, algo, final, tile=2048):
    """a leftmost-first feed -> chosen records [(chunk, end relative to the chunk, key)]"""
    flat, offs, held = emul_stream_leftmost.stage(st, chunks, ids)
    chosen, xn = settle(f, st, flat, offs, held, ids, algo, final, tile)
    _commit(st, chunks, ids, flat, offs, xn, final)
    return [(h, e - held[h], k) for h, e, k in chosen.tolist()]


def replace_feed(f, st, chunks, ids, algo, final, rep, rep_off, tile=2048):
    """a replacing leftmost-first feed -> (output bytes, output offsets)"""
    L = st["L"]
    flat, offs, held = emul_stream_leftmost.stage(st, chunks, ids)
    chosen, xn = settle(f, st, flat, offs, held, ids, algo, final, tile)
    win = np.concatenate([flat[offs[h]:offs[h] + xn[h] * L] for h in range(len(chunks))]) if chunks else np.empty(0, np.uint8)
    woff = np.zeros(len(chunks) + 1, dtype=np.int64)
    np.cumsum(xn * L, out=woff[1:])
    out, out_off = emul_replace.replace(win, woff, chosen, f["key_len"], rep, rep_off, L, 4096)
    _commit(st, chunks, ids, flat, offs, xn, final)
    return out, out_off


def new_state(A, n_streams, words):
    if words is None:
        return emul_stream_leftmost._state(A, n_streams)
    return emul_stream_words.new_state(A, n_streams, True, words)


def _common(self, op, args):
    if "bits" in self._ss:
        return emul_stream_words._common(self, op, args)
    return emul_stream_leftmost._common(self, self._ss, op, args)


# ------------------------------------------------------------------ the Python layer on the restatement
def install(monkeypatch, tile: int = 2048, algo: str = "filter"):
    """The leftmost-first paths of Automaton._leftmost_host, Automaton._words_host, Replacer._run_host,
    StreamBatch._native and ReplaceStream._native -> the emulated scan + select_first (+ word flags, replacement passes,
    stream staging) at the given tile size."""
    from pyahocorasick_b200 import _native as N
    from pyahocorasick_b200 import automaton as am

    scan = emul.install(None, algo)
    real = {"_leftmost_host": am.Automaton._leftmost_host, "_words_host": am.Automaton._words_host,
            "_run_host": am.Replacer._run_host, "stream": am.StreamBatch._native, "replace": am.ReplaceStream._native}

    def chosen_of(A, flat, offsets, n_hay, stride, algo_, narrow, words):
        f = A.flat(narrow=narrow)
        full = scan(A, flat, offsets, n_hay, stride, algo=algo_, sort=False, narrow=narrow)
        full = full[np.random.default_rng(len(full)).permutation(len(full))]            # any order
        kl = np.asarray(f["key_len"], dtype=np.int64)
        if words is not None:
            full, kl = emul_words._filtered(A, flat, offsets, n_hay, stride, narrow, full, words)
        return select_first(_raw(full), kl, int(kl.max()) if len(kl) else 0, tile), kl

    def fake_leftmost_host(self, flat, offsets, n_hay, stride_bytes, algo_, device, narrow, select=N.SELECT_LONGEST):
        if select == N.SELECT_LONGEST:
            return real["_leftmost_host"](self, flat, offsets, n_hay, stride_bytes, algo_, device, narrow)
        if self.flat(narrow=narrow) is None:
            return np.empty(0, dtype=N.MATCH_DTYPE)
        return _records(chosen_of(self, flat, offsets, n_hay, stride_bytes, algo_, narrow, None)[0])

    def fake_words_host(self, flat, offsets, n_hay, stride_bytes, algo_, sort, device, narrow, words, leftmost,
                        select=N.SELECT_LONGEST):
        if not leftmost or select == N.SELECT_LONGEST:
            return real["_words_host"](self, flat, offsets, n_hay, stride_bytes, algo_, sort, device, narrow, words, leftmost)
        if self.flat(narrow=narrow) is None:
            return np.empty(0, dtype=N.MATCH_DTYPE)
        return _records(chosen_of(self, flat, offsets, n_hay, stride_bytes, algo_, narrow, words)[0])

    def fake_run_host(self, flat, offs, n, narrow, algo_, words=None):
        if self._select == N.SELECT_LONGEST:
            return real["_run_host"](self, flat, offs, n, narrow, algo_, *(() if words is None else (words,)))
        A = self._A
        if A.flat(narrow=narrow) is None:
            return flat.copy(), offs.copy()
        chosen, kl = chosen_of(A, flat, offs, n, 0, algo_, narrow, words)
        rep, rep_off = self._tables[narrow]
        return emul_replace.replace(flat, offs, chosen, kl, rep, rep_off, 1 if narrow else A._L, 4096)

    def fake_stream(self, op, *args):
        if not self.leftmost_first:
            return real["stream"](self, op, *args)
        if op in ("new_leftmost", "new_words"):
            return new_state(self._A, self.n_streams, self._words)
        done, res = _common(self, op, args)
        if done:
            return res
        assert op == "feed_leftmost"
        kind, data, offs, n, stride, ids, final = args
        assert kind == "host"
        recs = feed(self._A.flat(), self._ss, emul_stream_leftmost._chunks(data, offs, n, stride), ids,
                    algo if self._algo == "auto" else self._algo, final, tile)
        return _records(recs)

    def fake_replace(self, op, *args):
        if self._R._select == N.SELECT_LONGEST:
            return real["replace"](self, op, *args)
        if op == "new":
            return new_state(self._A, self.n_streams, self._words)
        done, res = _common(self, op, args)
        if done:
            return res
        kind, data, offs, n, stride, ids, final = args
        assert kind == "host"
        rep, rep_off = self._R._tables[False]
        return replace_feed(self._A.flat(), self._ss, emul_stream_leftmost._chunks(data, offs, n, stride), ids,
                            algo if self._algo == "auto" else self._algo, final, rep, rep_off, tile)

    monkeypatch.setattr(am.Automaton, "_leftmost_host", fake_leftmost_host)
    monkeypatch.setattr(am.Automaton, "_words_host", fake_words_host)
    monkeypatch.setattr(am.Replacer, "_run_host", fake_run_host)
    monkeypatch.setattr(am.StreamBatch, "_native", fake_stream)
    monkeypatch.setattr(am.ReplaceStream, "_native", fake_replace)
