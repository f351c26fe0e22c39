#!/usr/bin/env python3
"""Whole-word stream feeds (DESIGN 4.15) against the feeds without words, batch resident in HBM.

    python tools/time_stream_words.py [--config C2 C3 C5 C4] [--steps 50] [--warmup 3] [--words abcdefghijklmnopqrstuvwxyz]

As tools/time_stream_leftmost.py does, each configuration's batch is fed as the next chunk of every stream (C2: 1 M
streams x 256 B; C4: 64 streams x 16 MiB), warmup + steps times in a row, so that every feed after the first has letters
held back.  Each step times, alternating, the find_all feed (acb_streams_feed_device), the leftmost feed
(acb_streams_feed_leftmost_device) and the replacing feed (acb_streams_replace_device) of plain batches, then the same
three on whole-word batches (acb_streams_new_words; acb_streams_feed_words_device for find_all), each with CUDA events
around the whole call.  The word set is --words (the lowercase letters by default: on the alphanumeric C2 / C5 text about
a third of the planted keys are whole words).  A second pass with the library's kernel timing on gives the stage split
(medians; for the find_all word feed "selection" is the record sort).  Prints one JSON line per configuration, with the
card's name, power limit and SM clock read in the same run."""
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
from pyahocorasick_b200.automaton import _word_bits  # noqa: E402


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


KINDS = ("find_all", "leftmost", "replace", "w_find_all", "w_leftmost", "w_replace")


def run(config, steps, warmup, words):
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
    out_cap = total * 5 // 4 + (1 << 20)
    r_out = torch.empty(out_cap, dtype=torch.uint8, device="cuda")
    r_off = torch.empty(n + 1, dtype=torch.int64, device="cuda")
    r_tot = torch.zeros(1, dtype=torch.int64, device="cuda")
    bits, n_bits = _word_bits(("bytes", words), 1)
    handles = {}
    for kind in KINDS:
        ss = ctypes.c_void_p()
        if kind == "find_all":
            N.check(L.acb_streams_new(tb, n, 0, ctypes.byref(ss)))
        elif kind.startswith("w_"):
            N.check(L.acb_streams_new_words(tb, n, int(kind != "w_find_all"), N.ptr(bits) if n_bits else None, n_bits,
                                            ctypes.byref(ss)))
        else:
            N.check(L.acb_streams_new_leftmost(tb, n, ctypes.byref(ss)))
        handles[kind] = ss

    def feed(kind):
        ss = handles[kind]
        base = kind[2:] if kind.startswith("w_") else kind
        if kind == "find_all":
            N.check(L.acb_streams_feed_device(ss, tb, d.data_ptr(), total, None, n, stride, None, d_out.data_ptr(), cap,
                                              d_cnt.data_ptr(), stream, algo))
        elif kind == "w_find_all":
            N.check(L.acb_streams_feed_words_device(ss, tb, d.data_ptr(), total, None, n, stride, None, 0, d_out.data_ptr(),
                                                    cap, d_cnt.data_ptr(), stream, algo))
        elif base == "leftmost":
            N.check(L.acb_streams_feed_leftmost_device(ss, tb, d.data_ptr(), total, None, n, stride, None, 0, d_out.data_ptr(),
                                                       cap, d_cnt.data_ptr(), stream, algo))
        else:
            N.check(L.acb_streams_replace_device(ss, r, tb, d.data_ptr(), total, None, n, stride, None, 0, r_off.data_ptr(),
                                                 r_out.data_ptr(), out_cap, r_tot.data_ptr(), stream, algo))

    for _ in range(warmup):
        for k in KINDS:
            feed(k)
    torch.cuda.synchronize()
    ms = {k: [] for k in KINDS}
    counts = {}
    for _ in range(steps):
        for k in KINDS:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            feed(k)
            b.record()
            torch.cuda.synchronize()
            ms[k].append(a.elapsed_time(b))
            counts[k] = int(r_tot.item()) if k.endswith("replace") else int(d_cnt.item())
    assert all(counts[k] <= (out_cap if k.endswith("replace") else cap) for k in KINDS)
    L.acb_set_kernel_timing(1)
    timed = ("leftmost", "w_find_all", "w_leftmost", "w_replace")
    stages = {k: [] for k in timed}
    sl = (ctypes.c_float * 6)()
    for _ in range(min(steps, 20)):
        for k in timed:
            feed(k)
            torch.cuda.synchronize()
            N.check(L.acb_last_stream_leftmost_ms(sl, 6))
            stages[k].append(list(sl))
    L.acb_set_kernel_timing(0)
    for ss in handles.values():
        L.acb_streams_free(ss)
    names = ["stage", "scan", "filter", "selection", "window", "commit"]
    split = {k: {nm: med([s[i] for s in v]) for i, nm in enumerate(names) if k.endswith("replace") or nm != "window"}
             for k, v in stages.items()}
    feed_ms = {f"{k}_feed_ms": med(v) for k, v in ms.items()}
    return {"config": config, "n_streams": n, "chunk_bytes": stride, "tail_letters": int(A.get_stats()["longest_word"]) - 1,
            "words": words.decode("latin-1"), **feed_ms,
            "w_leftmost_over_leftmost": round(feed_ms["w_leftmost_feed_ms"] / feed_ms["leftmost_feed_ms"], 3),
            "w_find_all_over_leftmost": round(feed_ms["w_find_all_feed_ms"] / feed_ms["leftmost_feed_ms"], 3),
            "stages_ms": split, "records_last_feed": {k: counts[k] for k in KINDS if not k.endswith("replace")}, **card()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", nargs="+", default=["C2", "C3", "C5", "C4"])
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--words", default="abcdefghijklmnopqrstuvwxyz")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_stream_words.py needs a CUDA device")
    for c in args.config:
        print(json.dumps(run(c, args.steps, args.warmup, args.words.encode("latin-1"))), flush=True)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
