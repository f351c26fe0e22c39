"""Test-only restatement of the leftmost-longest replacement (acb_replace_device) in numpy, for the CPU suite, pass by
pass as the device runs it: the offsets pass (shifts, per-record positions, haystack offsets) and the write pass over
tiles of `tile` output bytes, each cut into 16-byte chunks that are either inside one segment or assembled byte by byte.
`definition` is the rule the tests pin, stated directly.  `install` routes Replacer._run_host through the restatement on
top of the emulated scan (tests/emul.py) and selection (tests/emul_leftmost.py)."""
from __future__ import annotations

import numpy as np

import emul_leftmost


def definition(hay, chosen, key_len, rep):
    """one haystack (a sequence of letters) with its chosen matches [(end, key)] (end ascending) replaced by rep[key]"""
    out, p = [], 0
    for end, key in chosen:
        s = end - key_len[key] + 1
        out += list(hay[p:s]) + list(rep[key])
        p = end + 1
    return out + list(hay[p:])


def offsets_pass(chosen, key_len, rep_off, L, in_off, total_bytes):
    """chosen (n, 3) records (hay, end, key) in haystack order -> (out_off[n_hay+1], P, E, IE, RS)"""
    chosen = np.asarray(chosen, dtype=np.int64).reshape(-1, 3)
    key_len, rep_off, in_off = (np.asarray(x, dtype=np.int64) for x in (key_len, rep_off, in_off))
    hay, end, key = chosen[:, 0], chosen[:, 1], chosen[:, 2]
    ln, rl = key_len[key], rep_off[key + 1] - rep_off[key]
    D = np.zeros(len(chosen) + 1, dtype=np.int64)
    np.cumsum(rl - ln * L, out=D[1:])
    S = in_off[hay] + (end - ln + 1) * L
    P = S + D[:-1]
    lo = np.searchsorted(hay, np.arange(len(in_off)), side="left")
    base = in_off.copy()
    base[-1] = total_bytes
    return base + D[lo], P, P + rl, S + ln * L, rep_off[key]


def _find(P, lo, hi, o):
    """last j in [lo, hi] with P[j] <= o, or lo - 1 (acb_rp_write_kernel's binary search)"""
    while lo <= hi:
        mid = (lo + hi) >> 1
        if P[mid] <= o:
            lo = mid + 1
        else:
            hi = mid - 1
    return hi


def write_pass(hay, rep, P, E, IE, RS, total, tile):
    """the output bytes: tiles of `tile` bytes, the records of tile t are ts[t] .. ts[t+1]; 16-byte chunks in one
    segment are copied as a block, the others byte by byte"""
    hay, rep = np.asarray(hay, dtype=np.uint8), np.asarray(rep, dtype=np.uint8)
    P, E, IE, RS = (np.asarray(x, dtype=np.int64) for x in (P, E, IE, RS))
    out = np.full(total, 0xAA, dtype=np.uint8)
    n_tiles = -(-total // tile)
    ts = [_find(P, 0, len(P) - 1, t * tile) for t in range(n_tiles + 1)]
    for t in range(n_tiles):
        lo, hi = max(ts[t], 0), ts[t + 1]
        for c in range(t * tile, min((t + 1) * tile, total), 16):
            ce = min(c + 16, (t + 1) * tile, total)
            k = _find(P, lo, hi, c)
            in_rep = k >= lo and c < E[k]
            if in_rep and ce <= E[k]:
                x = RS[k] + c - P[k]
                out[c:ce] = rep[x:x + ce - c]
                continue
            if not in_rep and (k == hi or ce <= P[k + 1]):
                x = IE[k] + c - E[k] if k >= lo else c
                out[c:ce] = hay[x:x + ce - c]
                continue
            for o in range(c, ce):
                k = _find(P, max(k, lo), hi, o)
                if k >= lo and o < E[k]:
                    out[o] = rep[RS[k] + o - P[k]]
                else:
                    out[o] = hay[IE[k] + o - E[k] if k >= lo else o]
    return out


def replace(hay, in_off, chosen, key_len, rep, rep_off, L, tile):
    """both passes: (output bytes, output offsets)"""
    out_off, P, E, IE, RS = offsets_pass(chosen, key_len, rep_off, L, in_off, len(hay))
    return write_pass(hay, rep, P, E, IE, RS, int(out_off[-1]), tile), out_off


def install(monkeypatch, tile: int = 4096, algo: str = "filter"):
    """Replacer._run_host -> the emulated scan (unsorted) + emul_leftmost.select + both passes at the given tile size"""
    import emul
    from pyahocorasick_b200 import automaton as am

    scan = emul.install(None, algo)

    def fake_run_host(self, flat, offs, n, narrow, algo_):
        A = self._A
        f = A.flat(narrow=narrow)
        if f is None:
            return flat.copy(), offs.copy()
        full = scan(A, flat, offs, n, 0, algo=algo_, sort=False, narrow=narrow)
        raw = np.stack([full["hay_id"], full["end_index"], full["key_id"]], axis=1) if len(full) else np.empty((0, 3))
        kl = np.asarray(f["key_len"], dtype=np.int64)
        chosen = emul_leftmost.select(raw, kl, int(kl.max()) if len(kl) else 0)
        rep, rep_off = self._tables[narrow]
        return replace(flat, offs, chosen, kl, rep, rep_off, 1 if narrow else A._L, tile)

    monkeypatch.setattr(am.Replacer, "_run_host", fake_run_host)
