"""Test-only restatement of the white-space scans in numpy, for the CPU suite.  It replaces Automaton._scan_skip (every
find_all_batch(..., ignore_white_space=True)) and the skip stream batches of StreamBatch._native ("new_skip" and the
feeds of such a batch) with what the device does, stated plainly: drop the letters of the skip set from every haystack
or chunk, scan what is left with the emulated kernels (tests/emul.py, tests/emul_streams.py), and map every record's
end_index back through the positions of the kept letters.  The skip set itself is the package's (_skip_set)."""
from __future__ import annotations

import numpy as np

import emul
import emul_streams

_DT = {1: np.uint8, 2: np.dtype("<u2"), 4: np.dtype("<u4")}


def compact(raw: bytes, L: int, skip: np.ndarray):
    """(kept letters as bytes, original index of every kept letter)"""
    letters = np.frombuffer(raw, dtype=_DT[L])
    keep = ~np.isin(letters, skip)
    return letters[keep].tobytes(), np.nonzero(keep)[0]


def install(monkeypatch, algo="filter"):
    from pyahocorasick_b200 import _native as N
    from pyahocorasick_b200 import automaton as am

    emul.install(monkeypatch, algo)
    base = emul_streams.install(monkeypatch, algo)

    def fake_scan_skip(self, batch, algo_, sort, device):
        assert batch[0] == "host"
        _, flat, offs, n, stride, narrow = batch
        L = 1 if narrow else self._L
        skip = self._skip_set(narrow)
        raw = np.asarray(flat, dtype=np.uint8).tobytes()
        bounds = offs.tolist() if offs is not None else [h * stride for h in range(n + 1)]
        parts, maps = zip(*[compact(raw[bounds[h]:bounds[h + 1]], L, skip) for h in range(n)]) if n else ((), ())
        koff = np.zeros(n + 1, dtype=np.int64)
        np.cumsum([len(x) for x in parts], out=koff[1:])
        kflat = np.frombuffer(b"".join(parts), dtype=np.uint8)
        rec = self._scan_flat(kflat, koff, n, 0, algo=algo_, sort=sort, device=device, narrow=narrow)
        rec = np.array(rec, dtype=N.MATCH_DTYPE)
        for i in range(len(rec)):
            rec[i]["end_index"] = maps[rec[i]["hay_id"]][rec[i]["end_index"]]
        return rec

    def fake_native(self, op, *args):
        if op == "new_skip":
            st = base(self, "new")
            st["skip"] = args[0]
            st["opos"] = np.zeros(self.n_streams, dtype=np.int64)
            return st
        st = self._ss
        if "skip" not in st:
            return base(self, op, *args)
        if op == "positions":
            return st["opos"].copy()
        if op == "reset":
            base(self, op, *args)
            st["opos"][slice(None) if args[0] is None else args[0]] = 0
            return None
        if op == "free":
            return None
        kind, data, offs, n, stride, ids, sort = args
        assert kind == "host"
        L = self._A._L
        raw = np.asarray(data, dtype=np.uint8).tobytes()
        bounds = offs.tolist() if offs is not None else [h * stride for h in range(n + 1)]
        parts = [compact(raw[bounds[h]:bounds[h + 1]], L, st["skip"]) for h in range(n)]
        a = algo if self._algo == "auto" else self._algo
        recs = emul_streams.feed(self._A.flat(), st, [p for p, _ in parts], ids, a, False)   # st["pos"]: kept letters
        for h in range(n):
            st["opos"][h if ids is None else int(ids[h])] += (bounds[h + 1] - bounds[h]) // L
        out = np.empty(len(recs), dtype=N.MATCH_DTYPE)
        for i, (h, e, k) in enumerate(recs):
            out[i] = (h, parts[h][1][e], k)
        return out

    monkeypatch.setattr(am.Automaton, "_scan_skip", fake_scan_skip)
    monkeypatch.setattr(am.StreamBatch, "_native", fake_native)
