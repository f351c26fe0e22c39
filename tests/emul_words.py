"""Test-only restatement of the whole-word filter (acb_word_filter_device) in numpy, for the CPU suite: the flag of every
record from its two neighbour letters and a word bitmap, then the stable compaction below a capacity (exclusive sum,
emit, count).  `definition` is the rule the tests pin, stated directly over per-haystack letters.  `install` routes the
whole-word host routes of the Python layer (Automaton._words_host, Replacer._run_host) through the restatement on top of
the emulated scan (tests/emul.py), selection (tests/emul_leftmost.py) and replacement (tests/emul_replace.py)."""
from __future__ import annotations

import numpy as np

import emul_leftmost
import emul_replace


def definition(hays, full, key_len, is_word):
    """hays: letters per haystack; full: [(hay, end, key)] -> the records whose start has no word letter before it and
    whose end has no word letter after it, inside the haystack, in the order of `full`"""
    out = []
    for h, e, k in full:
        hay = hays[h]
        s = e - key_len[k] + 1
        if (s == 0 or not is_word(hay[s - 1])) and (e == len(hay) - 1 or not is_word(hay[e + 1])):
            out.append((h, e, k))
    return out


def flags(flat: np.ndarray, offs, stride: int, L: int, rec: np.ndarray, key_len: np.ndarray, bits: np.ndarray, n_bits: int):
    """acb_ww_flag_kernel over (n, 3) records: one bool per record.  flat: the batch's bytes; offs: byte offsets or None
    (fixed stride)"""
    rec = np.asarray(rec, dtype=np.int64).reshape(-1, 3)
    if len(rec) == 0:
        return np.zeros(0, dtype=bool)
    h, end = rec[:, 0], rec[:, 1]
    start = end - np.asarray(key_len, dtype=np.int64)[rec[:, 2]] + 1
    if offs is not None:
        offs = np.asarray(offs, dtype=np.int64)
        b0, letters = offs[h], (offs[h + 1] - offs[h]) // L
    else:
        b0, letters = h * stride, np.full(len(rec), stride // L, dtype=np.int64)
    flat = np.asarray(flat, dtype=np.uint8)
    words = np.unpackbits(np.asarray(bits, dtype="<u4").view(np.uint8), bitorder="little")[:n_bits].astype(bool)

    def word_at(ok, letter):
        v = np.zeros(len(rec), dtype=np.int64)
        at = b0[ok] + letter[ok] * L
        for j in range(L):
            v[ok] |= flat[at + j].astype(np.int64) << (8 * j)
        w = np.zeros(len(rec), dtype=bool)
        inside = ok & (v < n_bits)
        w[inside] = words[v[inside]]
        return w

    return ~word_at(start > 0, start - 1) & ~word_at(end + 1 < letters, end + 1)


def compact(rec: np.ndarray, flag: np.ndarray, cap: int, count: int = 0):
    """exclusive sum of the flags, emit below cap from index `count` on, add the total: (stored records, new count)"""
    pos = np.cumsum(flag) - flag
    at = count + pos
    keep = flag & (at < cap)
    return np.asarray(rec)[keep], count + int(flag.sum())


def _filtered(A, flat, offs, n, stride, narrow, full, words):
    from pyahocorasick_b200 import _native as N
    from pyahocorasick_b200.automaton import _word_bits
    L = 1 if narrow else A._L
    bits, n_bits = _word_bits(words, L)
    kl = np.asarray(A.flat(narrow=narrow)["key_len"], dtype=np.int64)
    raw = np.stack([full["hay_id"], full["end_index"], full["key_id"]], axis=1) if len(full) else np.empty((0, 3), np.int64)
    kept, _ = compact(raw, flags(flat, offs, stride, L, raw, kl, bits, n_bits), len(raw))
    out = np.empty(len(kept), dtype=N.MATCH_DTYPE)
    for i, r in enumerate(kept.tolist()):
        out[i] = tuple(r)
    return out, kl


def install(monkeypatch, algo: str = "filter"):
    """Automaton._words_host and Replacer._run_host -> the emulated scan (unsorted) + flags + compaction, then the
    reference order, emul_leftmost.select, or emul_leftmost.select and emul_replace.replace"""
    import emul
    from pyahocorasick_b200 import _native as N
    from pyahocorasick_b200 import automaton as am

    scan = emul.install(None, algo)

    def fake_words_host(self, flat, offsets, n_hay, stride_bytes, algo_, sort, device, narrow, words, leftmost):
        if self.flat(narrow=narrow) is None:
            return np.empty(0, dtype=N.MATCH_DTYPE)
        full = scan(self, flat, offsets, n_hay, stride_bytes, algo=algo_, sort=False, narrow=narrow)
        full = full[np.random.default_rng(len(full)).permutation(len(full))]     # any order
        kept, kl = _filtered(self, flat, offsets, n_hay, stride_bytes, narrow, full, words)
        if leftmost:
            raw = np.stack([kept["hay_id"], kept["end_index"], kept["key_id"]], axis=1) if len(kept) else np.empty((0, 3))
            got = emul_leftmost.select(raw, kl, int(kl.max()) if len(kl) else 0)
            out = np.empty(len(got), dtype=N.MATCH_DTYPE)
            for i, r in enumerate(got.tolist()):
                out[i] = tuple(r)
            return out
        if sort:
            kept = kept[np.lexsort((-kl[kept["key_id"]], kept["end_index"], kept["hay_id"]))]
        return kept

    def fake_run_host(self, flat, offs, n, narrow, algo_, words=None):
        A = self._A
        f = A.flat(narrow=narrow)
        if f is None:
            return flat.copy(), offs.copy()
        full = scan(A, flat, offs, n, 0, algo=algo_, sort=False, narrow=narrow)
        kl = np.asarray(f["key_len"], dtype=np.int64)
        if words is not None:
            full, kl = _filtered(A, flat, offs, n, 0, narrow, full, words)
        raw = np.stack([full["hay_id"], full["end_index"], full["key_id"]], axis=1) if len(full) else np.empty((0, 3))
        chosen = emul_leftmost.select(raw, kl, int(kl.max()) if len(kl) else 0)
        rep, rep_off = self._tables[narrow]
        return emul_replace.replace(flat, offs, chosen, kl, rep, rep_off, 1 if narrow else A._L, 4096)

    monkeypatch.setattr(am.Automaton, "_words_host", fake_words_host)
    monkeypatch.setattr(am.Replacer, "_run_host", fake_run_host)
