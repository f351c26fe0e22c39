#!/usr/bin/env python3
"""Time the whole-word filter on device-resident batches.

    python tools/time_words.py [--reps 20] [--out DIR]

Workloads (pyahocorasick_b200.synth, C2's 10 k keys): C2 planted (1 M x 256 B) and C4 (64 x 16 MiB), each with the
default word set (re's \\w for bytes) and the empty one (every match kept).  For each, with the batch resident in HBM:
  scan_ms        acb_scan_device (filter kernel) into a device buffer: the library's CUDA events around the launch
  filter_ms      acb_word_filter_device on that full list: its CUDA events from the flags to the count (acb_last_words_ms)
  records        full list and kept records
  calls_ms       whole calls on the CUDA tensor, host clock to a device synchronise, results on the host (find_all and
                 leftmost) or on the device (replace): find_all_batch, find_leftmost_longest_batch and
                 Replacer.replace_batch, each without and with whole_words
Medians of `reps` calls after 3 warm-up calls.  Every workload's kept records are checked once against the definition
(numpy, over find_all_batch's records), and against find_all_batch(whole_words=...).  The card's name, power limit and
SM clocks are read in the same run.  Prints one JSON line (also written to DIR/words.json)."""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.time_leftmost import _card  # noqa: E402


def _definition(hay, rec, key_len, bits, n_bits):
    """the whole-word records among rec (n, 3) of a fixed-stride batch of 1-byte letters hay [n, stride]"""
    import numpy as np
    stride = hay.shape[1]
    flat = hay.reshape(-1)
    word = np.zeros(256, dtype=bool)
    word[:n_bits] = np.unpackbits(bits.view(np.uint8), bitorder="little")[:n_bits].astype(bool)
    h, end = rec[:, 0].astype(np.int64), rec[:, 1].astype(np.int64)
    start = end - key_len[rec[:, 2]] + 1
    left = start > 0
    right = end + 1 < stride
    bad = np.zeros(len(rec), dtype=bool)
    bad[left] |= word[flat[h[left] * stride + start[left] - 1]]
    bad[right] |= word[flat[h[right] * stride + end[right] + 1]]
    return rec[~bad]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to time")
    from pyahocorasick_b200 import _native as N
    from pyahocorasick_b200 import synth
    from pyahocorasick_b200.automaton import _word_bits
    lib = N.lib()
    stream = torch.cuda.current_stream().cuda_stream
    c2, c4 = synth.make("C2"), synth.make("C4")
    A = synth.build_automaton(c2.keys)                         # C4 uses C2's key set
    R = A.replacer({k: k.upper() for k in c2.keys})
    tb = A._ensure_table(0)
    key_len = np.asarray(A.flat()["key_len"], dtype=np.int64)
    res = {"card": _card(), "reps": a.reps}
    med = lambda xs: float(np.median(xs))                      # noqa: E731

    def wall(fn):
        out = []
        for r in range(3 + a.reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            if r >= 3:
                out.append((time.perf_counter() - t0) * 1e3)
        return med(out)

    for name, host in (("C2", c2.haystacks), ("C4", c4.haystacks)):
        d = torch.from_numpy(host).cuda()
        n, stride = d.shape
        cnt = torch.zeros(1, dtype=torch.int64, device="cuda")
        cap = 1 << 24
        full = torch.empty((cap, 3), dtype=torch.int32, device="cuda")
        kept_cnt = torch.zeros(1, dtype=torch.int64, device="cuda")
        out = torch.empty((cap, 3), dtype=torch.int32, device="cuda")
        for label, words in (("default", True), ("empty", b"")):
            bits, n_bits = _word_bits(A._words(words), 1)
            d_bits = torch.from_numpy(bits.view(np.int32).copy()).cuda() if n_bits else None
            rows = {"scan_ms": [], "filter_ms": []}
            ms = ctypes.c_float()
            lib.acb_set_kernel_timing(1)
            for r in range(3 + a.reps):
                cnt.zero_()
                N.check(lib.acb_scan_device(tb, d.data_ptr(), n * stride, None, n, stride, full.data_ptr(), cap, cnt.data_ptr(),
                                            stream, N.ALGO_FILTER))
                scan = lib.acb_last_kernel_ms()
                m = int(cnt.item())
                assert m <= cap
                kept_cnt.zero_()
                N.check(lib.acb_word_filter_device(tb, d.data_ptr(), n * stride, None, n, stride, full.data_ptr(), m,
                                                   d_bits.data_ptr() if n_bits else None, n_bits, out.data_ptr(), cap,
                                                   kept_cnt.data_ptr(), stream))
                N.check(lib.acb_last_words_ms(ctypes.byref(ms)))
                if r >= 3:
                    rows["scan_ms"].append(scan)
                    rows["filter_ms"].append(ms.value)
            lib.acb_set_kernel_timing(0)
            kept = int(kept_cnt.item())
            got = out[:kept].cpu().numpy()
            want = _definition(host, full[:m].cpu().numpy(), key_len, bits, n_bits)
            assert np.array_equal(got, want), (name, label)
            chk = A.find_all_batch(d, sort=False, whole_words=words)
            assert len(chk) == kept
            r = {k: med(v) for k, v in rows.items()}
            r["filter_over_scan"] = r["filter_ms"] / r["scan_ms"]
            r["records"] = {"full": m, "kept": kept}
            r["calls_ms"] = {
                "find_all": wall(lambda: A.find_all_batch(d)),
                "find_all_words": wall(lambda: A.find_all_batch(d, whole_words=words)),
                "leftmost": wall(lambda: A.find_leftmost_longest_batch(d)),
                "leftmost_words": wall(lambda: A.find_leftmost_longest_batch(d, whole_words=words)),
                "replace": wall(lambda: R.replace_batch(d)),
                "replace_words": wall(lambda: R.replace_batch(d, whole_words=words)),
            }
            res[f"{name}/{label}"] = r
        del d, full, out
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "words.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
