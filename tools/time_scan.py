#!/usr/bin/env python3
"""Kernel time of one scan of a bench configuration, with no check of the results: for the ACB_EXP_* timing builds
(DESIGN 4.1), which drop work on purpose and so cannot pass bench.py's own count check.

    ACB_LIB=.../libacb200_x.so python tools/time_scan.py [--config C2] [--steps 300] [--warmup 20]

Prints one JSON line: the mean CUDA-event time of a launch, in ms, and the match count of the last one.

    python tools/time_scan.py --streams [--config C2]

feeds the same batch, resident in HBM, as the next chunk of n_haystacks streams (acb_streams_feed_device), over and
over, so that every feed after the first has full tails to stitch; each step times one acb_scan_device of the batch
and one feed, alternating, and a torch.profiler pass splits the feed into its kernels (main scan, seam walk, commit)."""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from pyahocorasick_b200 import _native as N, synth  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C2")
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--streams", action="store_true", help="time stream-batch feeds against the plain scan")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_scan.py needs a CUDA device")
    w = synth.make(args.config, scale=1.0)
    A = synth.build_automaton(w.keys)
    L = N.lib()
    tb = A._ensure_table(0)
    n_hay, stride = w.haystacks.shape
    d_hay = torch.from_numpy(w.haystacks).cuda()
    cap = max(4 * n_hay, 1 << 20)
    d_out = torch.empty((cap, 3), dtype=torch.int32, device="cuda")
    d_cnt = torch.zeros(1, dtype=torch.int64, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream

    def scan():
        d_cnt.zero_()
        N.check(L.acb_scan_device(tb, d_hay.data_ptr(), int(w.haystacks.size), None, n_hay, stride, d_out.data_ptr(), cap,
                                  d_cnt.data_ptr(), stream, N.ALGOS["auto"]))

    if args.streams:
        return time_streams(args, w, A, L, tb, d_hay, d_out, d_cnt, cap, stream, scan)
    for _ in range(args.warmup):
        scan()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.steps)]
    for a, b in ev:
        a.record()
        scan()
        b.record()
    torch.cuda.synchronize()
    ms = [a.elapsed_time(b) for a, b in ev]
    print(json.dumps({"config": args.config, "lib": os.environ.get("ACB_LIB", "default"), "kernel_ms": float(np.mean(ms)),
                      "kernel_ms_median": float(np.median(ms)), "matches": int(d_cnt.item()),
                      "gpu": torch.cuda.get_device_name(0)}))


def time_streams(args, w, A, L, tb, d_hay, d_out, d_cnt, cap, stream, scan):
    import ctypes
    n_hay, stride = w.haystacks.shape
    ss = ctypes.c_void_p()
    N.check(L.acb_streams_new(tb, n_hay, 0, ctypes.byref(ss)))

    def feed():
        N.check(L.acb_streams_feed_device(ss, tb, d_hay.data_ptr(), int(w.haystacks.size), None, n_hay, stride, None,
                                          d_out.data_ptr(), cap, d_cnt.data_ptr(), stream, N.ALGOS["auto"]))

    for _ in range(args.warmup):
        scan()
        feed()
    torch.cuda.synchronize()
    ev = [[torch.cuda.Event(enable_timing=True) for _ in range(3)] for _ in range(args.steps)]
    for a, b, c in ev:
        a.record()
        scan()
        b.record()
        feed()
        c.record()
    torch.cuda.synchronize()
    feed_count = int(d_cnt.item())
    scan()
    torch.cuda.synchronize()
    scan_count = int(d_cnt.item())
    scan_ms = [a.elapsed_time(b) for a, b, _ in ev]
    feed_ms = [b.elapsed_time(c) for _, b, c in ev]
    parts = {}
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(20):
            feed()
        torch.cuda.synchronize()
    for e in prof.key_averages():
        name = e.key
        part = ("seam" if "acb_seam_kernel" in name else "commit" if "commit_kernel" in name else
                "main_scan" if ("pair_kernel" in name or "stream_kernel" in name or "dfa_kernel" in name) else "other")
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        parts[part] = parts.get(part, 0.0) + t / 1000.0 / 20
    pos = np.zeros(n_hay, dtype=np.int64)
    N.check(L.acb_streams_positions(ss, N.ptr(pos), n_hay))
    L.acb_streams_free(ss)
    dev = torch.cuda.current_device()
    print(json.dumps({"config": args.config, "mode": "streams", "n_streams": n_hay, "chunk_bytes": stride,
                      "tail_letters": int(A.get_stats()["longest_word"]) - 1,
                      "scan_ms": float(np.mean(scan_ms)), "scan_ms_median": float(np.median(scan_ms)),
                      "feed_ms": float(np.mean(feed_ms)), "feed_ms_median": float(np.median(feed_ms)),
                      "feed_parts_ms": {k: round(v, 4) for k, v in parts.items()},
                      "scan_matches": scan_count, "feed_matches": feed_count, "capacity": cap,
                      "feeds_per_stream": int(pos[0] // stride),
                      "gpu": torch.cuda.get_device_name(dev)}))


if __name__ == "__main__":
    main()
