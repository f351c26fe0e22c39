#!/usr/bin/env python3
"""Leftmost-longest stream feeds (DESIGN 4.13) against the find_all feed, batch resident in HBM.

    python tools/time_stream_leftmost.py [--config C2 C3 C5 C4] [--steps 50] [--warmup 3] [--kinds longest,first]

As tools/time_scan.py --streams does, each configuration's batch is fed as the next chunk of every stream (C2: 1 M
streams x 256 B; C4: 64 streams x 16 MiB), warmup + steps times in a row, so that every feed after the first has
letters held back.  Each step times, alternating, one find_all feed (acb_streams_feed_device), one leftmost feed
(acb_streams_feed_leftmost_device) and one replacing feed (acb_streams_replace_device, every key replaced by a random
string of 0..19 bytes), each with CUDA events around the whole call (the feeds wait for their sizes inside the call).  A
second pass with the library's kernel timing on gives the stage split (medians): staging gather, scan, frontier filter,
selection, commit; for the replacing feed the window gather and the offsets and write passes.  A D2D copy of the chunk
bytes is timed in the same run.  Prints one JSON line per configuration, with the card's name, power limit and SM clock
read in the same run.  --kinds longest,first adds a leftmost-first feed and a leftmost-first replacing feed (batches of
acb_streams_new_leftmost_kind, a replacer of acb_replacer_new_kind) to the alternation, with their feed times, stage
splits and the ratios of their feed times to the leftmost-longest ones."""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from pyahocorasick_b200 import _native as N, synth  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, sm, sm_max = (x.strip() for x in q.split(","))
        return {"gpu": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}
    except Exception as e:                                       # the numbers are not worth much without these
        return {"gpu": torch.cuda.get_device_name(0), "card_query_error": str(e)}


def med(x):
    return round(float(np.median(x)), 4)


def run(config, steps, warmup, first=False):
    w = synth.make(config, scale=1.0)
    A = synth.build_automaton(w.keys)
    L = N.lib()
    tb = A._ensure_table(0)
    n, stride = w.haystacks.shape
    d = torch.from_numpy(w.haystacks).cuda()
    total = int(w.haystacks.size)
    stream = torch.cuda.current_stream().cuda_stream
    algo = N.ALGOS["auto"]
    cap = max(4 * n, 1 << 24)
    d_out = torch.empty((cap, 3), dtype=torch.int32, device="cuda")
    d_cnt = torch.zeros(1, dtype=torch.int64, device="cuda")
    rng = np.random.default_rng(1)
    keys = [k for k in A._key_objs if k is not None]
    R = A.replacer({k: bytes(rng.integers(0x41, 0x5B, size=int(rng.integers(0, 20)), dtype=np.uint8)) for k in keys})
    r = R._replacer(tb, False, 0)
    r_first = None
    if first:
        r_first = ctypes.c_void_p()
        flat, offs = R._tables[False]
        N.check(L.acb_replacer_new_kind(tb, N.SELECT_FIRST, N.ptr(flat), flat.size, N.ptr(offs), len(offs) - 1, ctypes.byref(r_first)))
    kinds = ("find_all", "leftmost", "replace") + (("leftmost_first", "replace_first") if first else ())
    lm = [k for k in kinds if k != "find_all"]
    out_cap = total * 5 // 4 + (1 << 20)
    r_out = torch.empty(out_cap, dtype=torch.uint8, device="cuda")
    r_off = torch.empty(n + 1, dtype=torch.int64, device="cuda")
    r_tot = torch.zeros(1, dtype=torch.int64, device="cuda")
    handles = {}
    for kind in kinds:
        ss = ctypes.c_void_p()
        if kind == "find_all":
            N.check(L.acb_streams_new(tb, n, 0, ctypes.byref(ss)))
        elif kind.endswith("_first"):
            N.check(L.acb_streams_new_leftmost_kind(tb, n, N.SELECT_FIRST, None, -1, ctypes.byref(ss)))
        else:
            N.check(L.acb_streams_new_leftmost(tb, n, ctypes.byref(ss)))
        handles[kind] = ss

    def feed(kind):
        ss = handles[kind]
        if kind == "find_all":
            N.check(L.acb_streams_feed_device(ss, tb, d.data_ptr(), total, None, n, stride, None, d_out.data_ptr(), cap,
                                              d_cnt.data_ptr(), stream, algo))
        elif kind.startswith("leftmost"):
            N.check(L.acb_streams_feed_leftmost_device(ss, tb, d.data_ptr(), total, None, n, stride, None, 0, d_out.data_ptr(),
                                                       cap, d_cnt.data_ptr(), stream, algo))
        else:
            N.check(L.acb_streams_replace_device(ss, r_first if kind == "replace_first" else r, tb, d.data_ptr(), total, None, n, stride, None, 0, r_off.data_ptr(),
                                                 r_out.data_ptr(), out_cap, r_tot.data_ptr(), stream, algo))

    for _ in range(warmup):
        for k in kinds:
            feed(k)
    torch.cuda.synchronize()
    ms = {k: [] for k in kinds}
    counts = {}
    for _ in range(steps):
        for k in kinds:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            feed(k)
            b.record()
            torch.cuda.synchronize()
            ms[k].append(a.elapsed_time(b))
            counts[k] = int(r_tot.item()) if k.startswith("replace") else int(d_cnt.item())
    assert counts["find_all"] <= cap and counts["leftmost"] <= cap and counts["replace"] <= out_cap
    copy = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        d.clone()
        b.record()
        torch.cuda.synchronize()
        copy.append(a.elapsed_time(b))
    L.acb_set_kernel_timing(1)
    stages = {k: [] for k in lm}
    rp = []
    sl = (ctypes.c_float * 6)()
    rpm = (ctypes.c_float * 2)()
    for _ in range(min(steps, 20)):
        for k in lm:
            feed(k)
            torch.cuda.synchronize()
            N.check(L.acb_last_stream_leftmost_ms(sl, 6))
            stages[k].append(list(sl))
            if k == "replace":
                N.check(L.acb_last_replace_ms(rpm, 2))
                rp.append(list(rpm))
    L.acb_set_kernel_timing(0)
    pos = np.zeros(n, dtype=np.int64)
    N.check(L.acb_streams_positions(handles["leftmost"], N.ptr(pos), n))
    for ss in handles.values():
        L.acb_streams_free(ss)
    if r_first is not None:
        L.acb_replacer_free(r_first)
    names = ["stage", "scan", "filter", "selection", "window", "commit"]
    split = {k: {nm: med([s[i] for s in v]) for i, nm in enumerate(names) if k.startswith("replace") or nm != "window"}
             for k, v in stages.items()}
    split["replace"]["offsets_pass"] = med([x[0] for x in rp])
    split["replace"]["write_pass"] = med([x[1] for x in rp])
    extra = {}
    if first:
        extra = {"leftmost_first_feed_ms": med(ms["leftmost_first"]), "replace_first_feed_ms": med(ms["replace_first"]),
                 "first_over_longest_feed": round(float(np.median(ms["leftmost_first"]) / np.median(ms["leftmost"])), 4),
                 "first_over_longest_replace": round(float(np.median(ms["replace_first"]) / np.median(ms["replace"])), 4),
                 "records_leftmost_first_last_feed": counts["leftmost_first"]}
    return {"config": config, "n_streams": n, "chunk_bytes": stride, "tail_letters": int(A.get_stats()["longest_word"]) - 1,
            "feeds_per_stream": int(pos[0] // stride),
            "find_all_feed_ms": med(ms["find_all"]), "leftmost_feed_ms": med(ms["leftmost"]), "replace_feed_ms": med(ms["replace"]),
            "d2d_copy_ms": med(copy), "stages_ms": split,
            "records_find_all": counts["find_all"], "records_leftmost_last_feed": counts["leftmost"],
            "output_bytes_last_feed": counts["replace"], **extra, **card()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", nargs="+", default=["C2", "C3", "C5", "C4"])
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--kinds", default="longest", choices=["longest", "longest,first"])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_stream_leftmost.py needs a CUDA device")
    for c in args.config:
        print(json.dumps(run(c, args.steps, args.warmup, args.kinds == "longest,first")), flush=True)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
