#!/usr/bin/env python3
"""Time the leftmost-longest selection stage by stage on device-resident batches.

    python tools/time_leftmost.py [--reps 20] [--out DIR] [--kinds longest,first]

Workloads (pyahocorasick_b200.synth, C2's 10 k keys): C2 planted (1 M x 256 B), C4 (64 x 16 MiB), and C4's bytes as
one haystack of 1 GiB.  For each, with the batch resident in HBM:
  scan_ms        acb_scan_device (filter kernel) into a device buffer: the library's CUDA events around the launch
  sort_ms ...    acb_leftmost_longest_device on that full list, CUDA events between its stages (acb_last_leftmost_ms):
                 re-key/sort, candidates, successor, chain, emit
  select_ms      the sum of the five stages
  records        full list and chosen records
Medians of `reps` calls after 3 warm-up calls.  As context for the one-lane-per-haystack path, `long_ms` is one
acb_scan_device with ACB_ALGO_LONG (find_long_batch's kernel) on C4.  Every workload's chosen
records are checked once against find_leftmost_longest_batch with algo="dfa".  The card's name, power limit and SM
clocks are read in the same run.  Prints one JSON line (also written to DIR/leftmost.json).

--kinds longest,first times acb_leftmost_first_device too, alternating with the leftmost-longest call on the same full
list in every repetition; each workload then also has "first" (its stages, select_ms and records, checked against
find_leftmost_first_batch) and "first_over_longest" (the ratio of the select_ms medians)."""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

STAGES = ("sort_ms", "candidates_ms", "successor_ms", "chain_ms", "emit_ms")


def _card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), [x.strip() for x in out.split(",")]))
    except Exception as e:                                      # the timings stand without it; say so
        return {"error": str(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    ap.add_argument("--kinds", default="longest", choices=["longest", "longest,first"])
    a = ap.parse_args()
    first = a.kinds == "longest,first"
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to time")
    from pyahocorasick_b200 import _native as N
    from pyahocorasick_b200 import synth
    lib = N.lib()
    stream = torch.cuda.current_stream().cuda_stream
    c2, c4 = synth.make("C2"), synth.make("C4")
    A = synth.build_automaton(c2.keys)                         # C4 uses C2's key set
    tb = A._ensure_table(0)
    work = {"C2": c2.haystacks, "C4": c4.haystacks, "1GiB": c4.haystacks.reshape(1, -1)}
    res = {"card": _card(), "reps": a.reps}
    med = lambda xs: float(np.median(xs))                      # noqa: E731
    for name, host in work.items():
        d = torch.from_numpy(host).cuda()
        n, stride = d.shape
        cnt = torch.zeros(1, dtype=torch.int64, device="cuda")
        cap = 1 << 24
        full = torch.empty((cap, 3), dtype=torch.int32, device="cuda")
        sel_cnt = torch.zeros(1, dtype=torch.int64, device="cuda")
        out = torch.empty((cap, 3), dtype=torch.int32, device="cuda")
        ms = (ctypes.c_float * 5)()
        rows = {k: [] for k in ("scan_ms",) + STAGES}
        rows_first = {k: [] for k in STAGES}
        first_cnt = torch.zeros(1, dtype=torch.int64, device="cuda")
        lib.acb_set_kernel_timing(1)
        for r in range(3 + a.reps):
            cnt.zero_()
            N.check(lib.acb_scan_device(tb, d.data_ptr(), n * stride, None, n, stride, full.data_ptr(), cap, cnt.data_ptr(),
                                        stream, N.ALGO_FILTER))
            scan = lib.acb_last_kernel_ms()
            m = int(cnt.item())
            assert m <= cap
            sel_cnt.zero_()
            N.check(lib.acb_leftmost_longest_device(tb, full.data_ptr(), m, n, stride, out.data_ptr(), cap, sel_cnt.data_ptr(), stream))
            N.check(lib.acb_last_leftmost_ms(ms, 5))
            if r >= 3:
                rows["scan_ms"].append(scan)
                for k, v in zip(STAGES, ms):
                    rows[k].append(v)
            if first:
                first_cnt.zero_()
                N.check(lib.acb_leftmost_first_device(tb, full.data_ptr(), m, n, stride, full[m:].data_ptr(), cap - m,
                                                      first_cnt.data_ptr(), stream))
                N.check(lib.acb_last_leftmost_ms(ms, 5))
                if r >= 3:
                    for k, v in zip(STAGES, ms):
                        rows_first[k].append(v)
        lib.acb_set_kernel_timing(0)
        chosen = int(sel_cnt.item())
        got = out[:chosen].cpu().numpy()
        chk = A.find_leftmost_longest_batch(d, algo="dfa")
        assert np.array_equal(got[:, 0], chk.hay_id) and np.array_equal(got[:, 1], chk.end_index) and np.array_equal(got[:, 2], chk.key_id)
        r = {k: med(v) for k, v in rows.items()}
        r["select_ms"] = sum(r[k] for k in STAGES)
        r["records"] = {"full": m, "chosen": chosen}
        if first:
            n_first = int(first_cnt.item())
            assert n_first <= cap - m
            chk = A.find_leftmost_first_batch(d, algo="dfa")
            got = full[m:m + n_first].cpu().numpy()
            assert np.array_equal(got[:, 0], chk.hay_id) and np.array_equal(got[:, 1], chk.end_index) and np.array_equal(got[:, 2], chk.key_id)
            f = {k: med(v) for k, v in rows_first.items()}
            f["select_ms"] = sum(f[k] for k in STAGES)
            f["records"] = {"full": m, "chosen": n_first}
            r["first"] = f
            r["first_over_longest"] = f["select_ms"] / r["select_ms"]
        if name == "C4":                                       # one lane per haystack: one launch, seconds long
            lib.acb_set_kernel_timing(1)
            cnt.zero_()
            N.check(lib.acb_scan_device(tb, d.data_ptr(), n * stride, None, n, stride, full.data_ptr(), cap, cnt.data_ptr(),
                                        stream, N.ALGO_LONG))
            r["long_ms"] = lib.acb_last_kernel_ms()
            r["long_records"] = int(cnt.item())
            lib.acb_set_kernel_timing(0)
        res[name] = r
        del d, full, out
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "leftmost.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
