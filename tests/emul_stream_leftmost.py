"""Test-only restatement of a leftmost-longest stream feed (acb_streams_feed_leftmost_*, acb_streams_replace_*,
csrc/acb_device.cu) in Python, on the scans of tests/emul.py, the selection of tests/emul_leftmost.py and the
replacement passes of tests/emul_replace.py.  It replaces StreamBatch._native (for leftmost_longest batches) and
ReplaceStream._native, the methods through which the Python layer reaches the native batch, so that the CPU suite runs
both classes against it.

Per stream it keeps what the device keeps: the position and the held letters (pos - X of them, X the position up to which
everything is decided).  A feed stages held || chunk per chunk, scans the staged batch, keeps the records that start
before the frontier staged_len - T (all on a final feed), selects, computes the new X per chunk
(max(0, staged_len - T, last chosen end + 1), staged_len on a final feed) and commits.  A replacing feed rewrites the
windows [0, new X) of the staged haystacks.  An emulated feed never overflows.
"""
from __future__ import annotations

import numpy as np

import emul
import emul_leftmost
import emul_replace


def stage(st, chunks, ids):
    """held || chunk per chunk -> (flat uint8, byte offsets, held letters per chunk)"""
    L = st["L"]
    staged, held = [], []
    for h, c in enumerate(chunks):
        s = h if ids is None else int(ids[h])
        staged.append(st["held"][s] + c)
        held.append(len(st["held"][s]) // L)
    offs = np.zeros(len(staged) + 1, dtype=np.int64)
    np.cumsum([len(x) for x in staged], out=offs[1:])
    flat = np.frombuffer(b"".join(staged), dtype=np.uint8) if staged else np.empty(0, np.uint8)
    return flat, offs, held


def settle(f, st, flat, offs, algo, final):
    """scan, frontier filter, selection -> (chosen (n, 3) staged coordinates, new X per chunk in staged letters)"""
    L, T, kl = st["L"], st["T"], np.asarray(f["key_len"], dtype=np.int64)
    n = len(offs) - 1
    scan = emul.emul_dfa if algo == "dfa" else emul.emul_filter
    full = scan(f, flat, offs) if flat.size else []
    staged_len = np.diff(offs) // L
    settled = [r for r in full if final or r[1] - kl[r[2]] + 1 < staged_len[r[0]] - T]
    chosen = emul_leftmost.select(np.array(settled, dtype=np.int64).reshape(-1, 3), kl, int(kl.max()) if len(kl) else 0)
    last = np.full(n, -1, dtype=np.int64)
    for h, e, _ in chosen.tolist():
        last[h] = e
    xn = staged_len.copy() if final else np.maximum(np.maximum(staged_len - T, 0), last + 1)
    return chosen, xn


def commit(st, chunks, ids, flat, offs, xn, final):
    L = st["L"]
    for h, c in enumerate(chunks):
        s = h if ids is None else int(ids[h])
        st["held"][s] = b"" if final else flat[offs[h] + xn[h] * L:offs[h + 1]].tobytes()
        st["pos"][s] = 0 if final else st["pos"][s] + len(c) // L


def feed(f, st, chunks, ids, algo, final):
    """the leftmost feed -> chosen records [(chunk, end relative to the chunk, key)]"""
    flat, offs, held = stage(st, chunks, ids)
    chosen, xn = settle(f, st, flat, offs, algo, final)
    commit(st, chunks, ids, flat, offs, xn, final)
    return [(h, e - held[h], k) for h, e, k in chosen.tolist()]


def replace_feed(f, st, chunks, ids, algo, final, rep, rep_off, tile=4096):
    """the replacing feed -> (output bytes, output offsets)"""
    L = st["L"]
    flat, offs, _ = stage(st, chunks, ids)
    chosen, xn = settle(f, st, flat, offs, algo, final)
    win = np.concatenate([flat[offs[h]:offs[h] + xn[h] * L] for h in range(len(chunks))]) if chunks else np.empty(0, np.uint8)
    woff = np.zeros(len(chunks) + 1, dtype=np.int64)
    np.cumsum(xn * L, out=woff[1:])
    out, out_off = emul_replace.replace(win, woff, chosen, f["key_len"], rep, rep_off, L, tile)
    commit(st, chunks, ids, flat, offs, xn, final)
    return out, out_off


def _state(A, n_streams):
    f = A.flat()
    L = f["letter_bytes"]
    return {"L": L, "T": max(f["max_key_bytes"] // L - 1, 0), "pos": np.zeros(n_streams, dtype=np.int64),
            "held": [b""] * n_streams}


def _common(self, st, op, args):
    """free / reset / positions on the emulated state; None when op is a feed"""
    if op == "free":
        return True, None
    if op == "reset":
        ids, = args
        for s in (range(self.n_streams) if ids is None else ids.tolist()):
            st["pos"][s], st["held"][s] = 0, b""
        return True, None
    if op == "positions":
        return True, st["pos"].copy()
    return False, None


def _chunks(data, offs, n, stride):
    raw = np.asarray(data, dtype=np.uint8).tobytes()
    bounds = offs.tolist() if offs is not None else [h * stride for h in range(n + 1)]
    return [raw[bounds[h]:bounds[h + 1]] for h in range(n)]


def install(monkeypatch, algo="filter", tile=4096):
    """Route StreamBatch._native (leftmost_longest batches) and ReplaceStream._native through the emulation."""
    from pyahocorasick_b200 import _native as N
    from pyahocorasick_b200 import automaton as am

    real = am.StreamBatch._native

    def fake_stream(self, op, *args):
        if not self.leftmost_longest:
            return real(self, op, *args)
        if op == "new_leftmost":
            return _state(self._A, self.n_streams)
        done, res = _common(self, self._ss, op, args)
        if done:
            return res
        assert op == "feed_leftmost"
        kind, data, offs, n, stride, ids, final = args
        assert kind == "host"
        recs = feed(self._A.flat(), self._ss, _chunks(data, offs, n, stride), ids,
                    algo if self._algo == "auto" else self._algo, final)
        out = np.empty(len(recs), dtype=N.MATCH_DTYPE)
        for i, r in enumerate(recs):
            out[i] = r
        return out

    def fake_replace(self, op, *args):
        if op == "new":
            return _state(self._A, self.n_streams)
        done, res = _common(self, self._ss, op, args)
        if done:
            return res
        kind, data, offs, n, stride, ids, final = args
        assert kind == "host"
        rep, rep_off = self._R._tables[False]
        return replace_feed(self._A.flat(), self._ss, _chunks(data, offs, n, stride), ids,
                            algo if self._algo == "auto" else self._algo, final, rep, rep_off, tile)

    monkeypatch.setattr(am.StreamBatch, "_native", fake_stream)
    monkeypatch.setattr(am.ReplaceStream, "_native", fake_replace)
