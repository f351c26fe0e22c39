#!/usr/bin/env python3
"""Kernel time of one scan of a bench configuration, with no check of the results: for the ACB_EXP_* timing builds
(DESIGN 4.1), which drop work on purpose and so cannot pass bench.py's own count check.

    ACB_LIB=.../libacb200_x.so python tools/time_scan.py [--config C2] [--steps 300] [--warmup 20]

Prints one JSON line: the mean CUDA-event time of a launch, in ms, and the match count of the last one."""
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


if __name__ == "__main__":
    main()
