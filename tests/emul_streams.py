"""Test-only restatement of a stream-batch feed (acb_streams_*, csrc/acb_device.cu) in pure Python, on the kernels
restated in tests/emul.py.  It replaces StreamBatch._native, the one method through which the Python layer reaches the
native stream batch, so that the CPU suite runs StreamBatch against it.

Per stream it keeps what the device keeps: the position, the tail (the last T = longest_word - 1 letters consumed,
fewer at the start) and, for iter_long batches, the walk state.  A feed is the main scan of every chunk by itself, plus
for each chunk the seam -- tail + the first min(T, n) letters of the chunk -- walked from the root (emul_dfa), of which
only the matches that start in the tail and end in the chunk count (end >= t and end - len + 1 < t, rebased to
end - t).  Long batches continue each stream's walk from its state (emul_long(init_state=...)).  Everything commits at
the end of the feed: an emulated feed never overflows.
"""
from __future__ import annotations

import numpy as np

import emul


def feed(f, st, chunks, ids, algo, long):
    """chunks: list of byte strings (whole letters).  Returns [(chunk index, end in the chunk, key id)] sorted as the
    device feed sorts them, and updates st ({"T", "pos", "tail", "state"}) in place."""
    L, T, kl = f["letter_bytes"], st["T"], f["key_len"]
    main = emul.emul_dfa if algo == "dfa" else emul.emul_filter
    recs, staged = [], []
    for h, c in enumerate(chunks):
        s = h if ids is None else int(ids[h])
        buf = np.frombuffer(c, dtype=np.uint8)
        n = len(c) // L
        if long:
            got, end = emul.emul_long(f, buf, np.array([0, len(c)]), init_state=st["state"][s], want_state=True)
            recs += [(h, e, k) for _, e, k in got]
            staged.append((s, n, None, end))
            continue
        if len(c):
            recs += [(h, e, k) for _, e, k in main(f, buf, np.array([0, len(c)]))]
        tail = st["tail"][s]
        t = len(tail) // L
        seam = tail + c[:min(T, n) * L]
        if t and len(seam) > len(tail):
            sb = np.frombuffer(seam, dtype=np.uint8)
            for _, e, k in emul.emul_dfa(f, sb, np.array([0, len(seam)])):
                if e >= t and e - int(kl[k]) + 1 < t:
                    recs.append((h, e - t, k))
        whole = tail + c
        staged.append((s, n, whole[len(whole) - min(T, t + n) * L:], None))
    for s, n, tail, state in staged:                            # the commit
        st["pos"][s] += n
        if tail is not None:
            st["tail"][s] = tail
        if state is not None:
            st["state"][s] = state
    recs.sort(key=lambda r: (r[0], r[1], -int(kl[r[2]])))
    return recs


def install(monkeypatch, algo="filter"):
    """Route StreamBatch._native through the emulation (CPU tests of the Python layer only)."""
    from pyahocorasick_b200 import _native as N
    from pyahocorasick_b200 import automaton as am

    def fake_native(self, op, *args):
        A = self._A
        if op == "new":
            f = A.flat()
            T = 0 if self.long else max(f["max_key_bytes"] // f["letter_bytes"] - 1, 0)
            return {"T": T, "pos": np.zeros(self.n_streams, dtype=np.int64), "tail": [b""] * self.n_streams,
                    "state": [0] * self.n_streams}
        st = self._ss
        if op == "free":
            return None
        if op == "reset":
            ids, = args
            for s in (range(self.n_streams) if ids is None else ids.tolist()):
                st["pos"][s], st["tail"][s], st["state"][s] = 0, b"", 0
            return None
        if op == "positions":
            return st["pos"].copy()
        kind, data, offs, n, stride, ids, sort = args
        assert kind == "host"
        raw = np.asarray(data, dtype=np.uint8).tobytes()
        bounds = offs.tolist() if offs is not None else [h * stride for h in range(n + 1)]
        chunks = [raw[bounds[h]:bounds[h + 1]] for h in range(n)]
        a = algo if self._algo == "auto" else self._algo
        recs = feed(A.flat(), st, chunks, ids, a, self.long)
        out = np.empty(len(recs), dtype=N.MATCH_DTYPE)
        for i, r in enumerate(recs):
            out[i] = r
        return out

    monkeypatch.setattr(am.StreamBatch, "_native", fake_native)
    return fake_native
