#!/usr/bin/env python3
"""Time keys / values / items with prefix and wildcard on the reference's published key set, per key and as one batch.

    python tools/time_select.py [--words 1000000] [--queries 1000000] [--reps 20] [--sample 3] [--out DIR]

Keys are the published benchmark's words (tools/time_lookup.py's generator: N random words of 3..32 characters over
[a-zA-Z0-9], bytes flavour, each stored with its index).  Two query sets: `prefix`, Q random 3-letter prefixes (no
wildcard: every key that starts with them), and `wildcard`, Q patterns of 3 random letters and two '?' with
how = MATCH_EXACT_LENGTH (keys of exactly 5 letters).  For each set it reports:
  select_batch_s / keys_batch_s   host clock around select_batch(list) / keys_batch(list), table and key ranges already
                                  on the device, median of 5 (keys_batch also maps ids to key objects)
  kernel_ms                       acb_select_device on device-resident patterns (both passes and the scan between them):
                                  CUDA events (the library's kernel timing), median of `reps` calls after 3 warm-up calls
  ids                             keys selected in all
and once: upload_key_ranges_s (acb_table_upload_key_ranges: the host walk and the copy), and per_key_keys_s /
reference_keys_s, list(keys(p)) per pattern on `sample` patterns of each set for the drop-in and the reference
(oracle/_ref, when it is built), in seconds per pattern -- measured, not extrapolated.  The card's name and power limit
are read in the same run.  Prints one JSON line (also written to DIR/select.json)."""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from time_lookup import _card, _clock, words_and_misses   # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--words", type=int, default=1_000_000)
    ap.add_argument("--queries", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--sample", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to time")
    import pyahocorasick_b200 as pkg
    from pyahocorasick_b200 import _native as N
    words, _ = words_and_misses(a.words)
    keys = [w.encode() for w in words]
    A = pkg.flavour("bytes").Automaton(pkg.STORE_INTS)
    for i, k in enumerate(keys):
        A.add_word(k, i)
    A.make_automaton()
    lib = N.lib()
    tb = A._ensure_table(0)
    res = {"workload": f"{a.words} keys of 3..32 chars over [a-zA-Z0-9] (bytes flavour); {a.queries} patterns per set"}
    res["upload_key_ranges_s"], _ = _clock(lambda: N.check(lib.acb_table_upload_key_ranges(tb, A._trie)))

    rng = np.random.default_rng(0)
    chars = np.frombuffer(b"abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789", dtype=np.uint8)
    sets = {"prefix": ([bytes(r) for r in rng.choice(chars, size=(a.queries, 3))], None, pkg.MATCH_EXACT_LENGTH),
            "wildcard": ([bytes(r) + b"??" for r in rng.choice(chars, size=(a.queries, 3))], b"?", pkg.MATCH_EXACT_LENGTH)}
    import oracle
    R = None
    if oracle.ref_available("bytes"):
        R = oracle.ref_module("bytes").Automaton(oracle.ref_module("bytes").STORE_INTS)
        for i, k in enumerate(keys):
            R.add_word(k, i)
        R.make_automaton()
    for name, (pats, w, how) in sets.items():
        out = {}
        A.select_batch(pats, w, how)                            # warm-up
        t, tk = [], []
        for _ in range(5):
            dt, (offs, kid) = _clock(lambda: A.select_batch(pats, w, how))
            t.append(dt)
            dt, got = _clock(lambda: A.keys_batch(pats, w, how))
            tk.append(dt)
        out["select_batch_s"], out["keys_batch_s"] = float(np.median(t)), float(np.median(tk))
        out["ids"] = int(offs[-1])
        sample = rng.integers(0, len(pats), size=a.sample).tolist()
        dt, want = _clock(lambda: [list(A.keys(pats[i], w, how)) for i in sample])
        out["per_key_keys_s"] = dt / len(sample)
        assert [got[i] for i in sample] == want, "keys_batch differs from the keys() loop"
        if R is not None:
            rargs = () if w is None else (w, how)               # the reference takes no None wildcard
            dt, ref = _clock(lambda: [list(R.values(pats[i], *rargs)) for i in sample])
            out["reference_keys_s"] = dt / len(sample)
            assert ref == [[A.get(k) for k in ks] for ks in want], "the reference and the drop-in disagree"
        # both passes and the scan on device-resident patterns
        flat = np.frombuffer(b"".join(pats), dtype=np.uint8).reshape(len(pats), -1)
        d = torch.from_numpy(flat.copy()).cuda()
        n, stride = d.shape
        d_offs = torch.empty(n + 1, dtype=torch.int64, device="cuda")
        d_total = torch.empty(1, dtype=torch.int64, device="cuda")
        d_kid = torch.empty(max(out["ids"], 1), dtype=torch.int32, device="cuda")
        stream = torch.cuda.current_stream().cuda_stream
        torch.cuda.synchronize()
        lib.acb_set_kernel_timing(1)
        ms = []
        try:
            for i in range(3 + a.reps):
                N.check(lib.acb_select_device(tb, d.data_ptr(), n * stride, None, n, stride, -1 if w is None else w[0],
                                              how, d_offs.data_ptr(), d_kid.data_ptr(), d_kid.numel(), d_total.data_ptr(),
                                              stream))
                if i >= 3:
                    ms.append(float(lib.acb_last_kernel_ms()))
        finally:
            lib.acb_set_kernel_timing(0)
        assert (d_kid[:out["ids"]].cpu().numpy() == kid).all()
        out["kernel_ms"] = {"median": float(np.median(ms)), "min": float(np.min(ms)), "max": float(np.max(ms)), "calls": a.reps}
        res[name] = out
    res["card"], res["power_limit"] = _card()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "select.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
