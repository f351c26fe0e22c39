"""Test-only restatement of acb_select_kernel in Python, for the CPU suite.  It replaces Automaton._select_host (the one
native call of select_batch / keys_batch / values_batch / items_batch on host batches) with the kernel's walk over the
flattened tables of A.flat() and the key ranges of A.key_ranges(): without a wildcard one walk down the goto table and
the run order[lo:lo+cnt]; with one, the rank-cursor walk of the kernel, children of a wildcard letter taken from the
child list by a binary search on lo, and a path of only PATH nodes kept (deeper parents found again from the deepest
kept one, as on the device)."""
from __future__ import annotations

import numpy as np

_ID_MASK = 0x3FFFFFFF
EXACT, AT_MOST, AT_LEAST = 0, 1, 2
PATH = 16                              # kSelectPath


def _letter_step(f, b: bytes, x: int) -> int:
    cls, goto = f["byte_class"], f["goto_cm"]
    for byte in b:
        nx = int(goto[cls[byte], x])
        if nx < 0:
            return -1
        x = nx & _ID_MASK
    return x


def walk(f: dict, kr: dict, pat: bytes, wildcard: int, how: int) -> list:
    """the ranks of one pattern's keys, in order"""
    L = f["letter_bytes"]
    key_of, lo, cnt, cp, child = f["key_of"], kr["lo"], kr["cnt"], kr["child_ptr"], kr["child"]
    m = len(pat) // L
    out = []
    if wildcard < 0:
        x = 0
        for j in range(m):
            x = _letter_step(f, pat[j * L:(j + 1) * L], x)
            if x < 0:
                return out
        return list(range(int(lo[x]), int(lo[x] + cnt[x])))
    path = [0] * PATH
    x, r, j = 0, 0, 0
    while True:
        xlo, xend = int(lo[x]), int(lo[x] + cnt[x])
        if j > 0 and xlo >= r and (how == AT_MOST or (how == EXACT and j == m)) and key_of[x] >= 0:
            out.append(xlo)
            r = xlo + 1
        c = -1
        if j == m:
            if how == AT_LEAST:
                out.extend(range(max(r, xlo), xend))
        else:
            b = pat[j * L:(j + 1) * L]
            if int.from_bytes(b, "little") == wildcard:
                kids = child[cp[x]:cp[x + 1]]
                a = int(np.searchsorted(lo[kids], r, side="right"))      # the first child with lo > r
                if a > 0 and lo[kids[a - 1]] + cnt[kids[a - 1]] > r:
                    c = int(kids[a - 1])
                elif a < len(kids):
                    c = int(kids[a])
            else:
                c = _letter_step(f, b, x)
                if c >= 0 and lo[c] + cnt[c] <= r:
                    c = -1
        if c < 0:
            r = max(r, xend)
            if j == 0:
                break
            j = min(j - 1, PATH - 1)
            x = path[j]
            continue
        x = c
        j += 1
        if j < PATH:
            path[j] = x
    return out


def select(f: dict, kr: dict, flat: np.ndarray, offsets, n: int, stride: int, wildcard: int, how: int):
    flat = np.asarray(flat, dtype=np.uint8).reshape(-1)
    raw = flat.tobytes()
    order = kr["order"]
    out_offs = np.zeros(n + 1, dtype=np.int64)
    ids = []
    for q in range(n):
        b0, b1 = (int(offsets[q]), int(offsets[q + 1])) if offsets is not None else (q * stride, (q + 1) * stride)
        ranks = walk(f, kr, raw[b0:b1], wildcard, how)
        ids.extend(int(order[k]) for k in ranks)
        out_offs[q + 1] = len(ids)
    return out_offs, np.asarray(ids, dtype=np.int32)


def install(monkeypatch):
    from pyahocorasick_b200 import automaton as am

    def fake_select_host(self, flat, offsets, n, stride_bytes, wildcard, how, device):
        return select(self.flat(), self.key_ranges(), flat, offsets, n, stride_bytes, wildcard, how)

    monkeypatch.setattr(am.Automaton, "_select_host", fake_select_host)
