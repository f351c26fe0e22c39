"""Test-only restatement of acb_lookup_kernel in numpy, for the CPU suite.  It replaces Automaton._lookup_host (the one
native call of exists_batch / match_batch / longest_prefix_batch / get_batch on host batches) with the kernel's walk over
the flattened tables of A.flat(): from the root, byte by byte through the column-major goto table, stopping at the first
missing edge; key_id = key_of[state] when every byte was consumed (and the query is not empty), prefix = whole letters
walked."""
from __future__ import annotations

import numpy as np

_ID_MASK = 0x3FFFFFFF                  # the device entries carry kTermBit; the host view does not, masking is harmless


def lookup(f: dict, flat: np.ndarray, offsets, n: int, stride: int):
    cls, goto, key_of, L = f["byte_class"], f["goto_cm"], f["key_of"], f["letter_bytes"]
    flat = np.asarray(flat, dtype=np.uint8).reshape(-1)
    key_id = np.empty(n, dtype=np.int32)
    prefix = np.empty(n, dtype=np.int32)
    for q in range(n):
        b0, b1 = (int(offsets[q]), int(offsets[q + 1])) if offsets is not None else (q * stride, (q + 1) * stride)
        s, i = 0, b0
        while i < b1:
            nx = int(goto[cls[flat[i]], s])
            if nx < 0:
                break
            s = nx & _ID_MASK
            i += 1
        key_id[q] = key_of[s] if i == b1 and b1 > b0 else -1
        prefix[q] = (i - b0) // L
    return key_id, prefix


def install(monkeypatch):
    from pyahocorasick_b200 import automaton as am

    def fake_lookup_host(self, flat, offsets, n, stride_bytes, device):
        return lookup(self.flat(), flat, offsets, n, stride_bytes)

    monkeypatch.setattr(am.Automaton, "_lookup_host", fake_lookup_host)
