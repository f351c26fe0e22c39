"""Test-only restatement of the leftmost-longest selection (acb_leftmost_longest_device) in numpy, for the CPU suite,
step by step as the device runs it: re-key by start and sort, keep the first record of every (hay, start) run, the
successor of every candidate, the chain marking over tiles of `tile` candidates with the merge-on-entry rule, emit.
`greedy` is the definition the tests pin, stated directly.  `install` routes Automaton._leftmost_host through the
restatement on top of the emulated scan (tests/emul.py)."""
from __future__ import annotations

import numpy as np


def greedy(recs, key_len):
    """The definition over a full match list [(hay, end, key)]: per haystack, p = 0; take the smallest start >= p, the
    longest match there, continue at its end + 1.  Returns the chosen records in haystack order, then end ascending."""
    by_hay = {}
    for h, e, k in recs:
        by_hay.setdefault(int(h), []).append((int(e) - int(key_len[k]) + 1, -int(key_len[k]), int(e), int(k)))
    out = []
    for h in sorted(by_hay):
        p = 0
        for s, _, e, k in sorted(by_hay[h]):
            if s >= p:
                out.append((h, e, k))
                p = e + 1
    return out


def select(rec: np.ndarray, key_len: np.ndarray, max_len: int, tile: int = 2048) -> np.ndarray:
    """The device's five steps on (n, 3) int records (hay, end, key) in any order -> the chosen records."""
    rec = np.asarray(rec, dtype=np.int64).reshape(-1, 3)
    key_len = np.asarray(key_len, dtype=np.int64)
    if len(rec) == 0:
        return np.empty((0, 3), dtype=np.int64)
    hay, end, key = rec[:, 0], rec[:, 1], rec[:, 2]
    ln = key_len[key]
    start = end - ln + 1
    # 1. re-key by start: hay | start | (max_len - len), a stable sort (the radix sort is stable)
    order = np.lexsort((max_len - ln, start, hay))
    hay, start, ln, srt = hay[order], start[order], ln[order], rec[order]
    # 2. candidates: the first record of every (hay, start) run
    first = np.ones(len(srt), dtype=bool)
    first[1:] = (hay[1:] != hay[:-1]) | (start[1:] != start[:-1])
    cand, chay, cstart, clen = srt[first], hay[first], start[first], ln[first]
    M = len(cand)
    # 3. successor: the first candidate of the same haystack with start >= start_i + len_i, searched in [i+1, i+len_i]
    nxt = np.full(M, -1, dtype=np.int64)
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
    # 4. chain marking over tiles
    chosen = chain(chay, nxt, max(max_len, 1), tile)
    # 5. emit: already in the final order
    return cand[chosen]


def chain(chay: np.ndarray, nxt: np.ndarray, W: int, tile: int) -> np.ndarray:
    """acb_ll_chain_kernel, tile by tile in claim order.  A tile publishes its exit early when it does not depend on
    the entry (a haystack starts in it, or every one of its first W candidates joins the speculative chain); the
    published exits are checked against the ones computed from the true entries."""
    M = len(chay)
    chosen = np.zeros(M, dtype=bool)
    status = {}
    for t in range((M + tile - 1) // tile):
        base = t * tile
        n = min(tile, M - base)
        head = [base + j == 0 or chay[base + j] != chay[base + j - 1] for j in range(n)]
        spec = np.zeros(n, dtype=bool)
        want, fh = base, n
        for j in range(n):
            if head[j]:
                want = base + j
                fh = min(fh, j)
            if want == base + j:
                spec[j] = True
                want = int(nxt[base + j])
        spec_exit = want
        dep = fh == n and n < W
        if fh == n and not dep:
            for j in range(W):
                e = base + j
                while base <= e < base + n and not spec[e - base]:
                    e = int(nxt[e])
                joined = base <= e < base + n and spec[e - base]
                if not joined and e != spec_exit:
                    dep = True
        fin = spec.copy()
        entry, ex = base, spec_exit
        if fh > 0 and t > 0:
            entry = status[t - 1]
        if entry != base:                                   # merge on entry
            e = entry
            while base <= e < base + fh and not spec[e - base]:
                fin[e - base] = True
                e = int(nxt[e])
            joined = base <= e < base + fh
            stop = e if joined else base + fh
            q = base
            while base <= q < stop:
                fin[q - base] = False
                q = int(nxt[q])
            if fh == n and not joined:
                ex = e
        if not dep:
            assert ex == spec_exit, (t, ex, spec_exit)    # an early exit must be the true one
        status[t] = ex
        chosen[base:base + n] = fin
    return chosen


def install(monkeypatch, tile: int = 2048, algo: str = "filter"):
    """Automaton._leftmost_host -> the emulated scan (unsorted) + select() at the given tile size."""
    import emul
    from pyahocorasick_b200 import _native as N
    from pyahocorasick_b200 import automaton as am

    scan = emul.install(None, algo)

    def fake_leftmost_host(self, flat, offsets, n_hay, stride_bytes, algo_, device, narrow):
        f = self.flat(narrow=narrow)
        if f is None:
            return np.empty(0, dtype=N.MATCH_DTYPE)
        full = scan(self, flat, offsets, n_hay, stride_bytes, algo=algo_, sort=False, narrow=narrow)
        rng = np.random.default_rng(len(full))
        full = full[rng.permutation(len(full))]            # any order
        raw = np.stack([full["hay_id"], full["end_index"], full["key_id"]], axis=1) if len(full) else np.empty((0, 3))
        kl = np.asarray(f["key_len"])
        got = select(raw, kl, int(kl.max()) if len(kl) else 0, tile)
        out = np.empty(len(got), dtype=N.MATCH_DTYPE)
        for i, r in enumerate(got.tolist()):
            out[i] = tuple(r)
        return out

    monkeypatch.setattr(am.Automaton, "_leftmost_host", fake_leftmost_host)
