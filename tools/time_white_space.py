"""Time find_all_batch(..., ignore_white_space=True) on a batch resident in HBM, split by kernel.

    python tools/time_white_space.py [--scale 1.0] [--rate 0.02] [--reps 20] [--out DIR]

The C2 planted batch (pyahocorasick_b200.synth) with a share `rate` of its bytes turned into spaces, as a uint8 CUDA
tensor.  Alternating within one run, each repetition times with CUDA events:
  skip   find_all_batch(d, ignore_white_space=True)   (compact, scan, remap, sort, records back)
  plain  find_all_batch(d)                            (the same bytes without the option)
  copy   a D2D cudaMemcpyAsync of the same bytes (torch copy_)
and a second alternating loop, with the library's kernel timing on (acb_set_kernel_timing: CUDA events around each
launch), times the compaction kernel, the scan of the compacted batch and the remap of every `skip` call
(acb_last_skip_ms, acb_last_kernel_ms), the scan kernel of every `plain` call and the copy.
The card's name and power limit are read in the same call.  Prints one JSON line (also written to DIR/white_space.json).
"""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in out.split(",")]
        return name, power
    except Exception as e:                                      # the timings stand without it; say so
        return f"unknown ({e})", "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--rate", type=float, default=0.02)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import numpy as np
    import torch
    from pyahocorasick_b200 import _native as N
    from pyahocorasick_b200 import synth
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to time")
    w = synth.make("C2", scale=a.scale)
    A = synth.build_automaton(w.keys)
    x = w.haystacks.copy()
    rng = np.random.default_rng(0)
    x[rng.random(x.shape) < a.rate] = ord(" ")
    d = torch.from_numpy(x).cuda()
    dst = torch.empty_like(d)
    nbytes = d.numel()

    def ev_time(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1)

    runs = {"skip": lambda: A.find_all_batch(d, ignore_white_space=True), "plain": lambda: A.find_all_batch(d),
            "copy": lambda: dst.copy_(d)}
    for fn in runs.values():                                    # warm-up: modules, scratch buffers, table upload
        fn()
    torch.cuda.synchronize()
    times = {k: [] for k in runs}
    for _ in range(a.reps):                                     # whole calls, kernel timing off
        for k, fn in runs.items():
            times[k].append(ev_time(fn))
    n_skip = len(A.find_all_batch(d, ignore_white_space=True))

    # kernels: the library's own CUDA events around each launch (acb_set_kernel_timing), again alternating with the
    # plain scan and the copy
    lib = N.lib()
    lib.acb_set_kernel_timing(1)
    cm, rm = ctypes.c_float(0), ctypes.c_float(0)
    kern = {"compact": [], "scan_compacted": [], "remap": [], "scan_plain": [], "copy": []}
    try:
        for _ in range(a.reps):
            runs["skip"]()
            N.check(lib.acb_last_skip_ms(ctypes.byref(cm), ctypes.byref(rm)))
            kern["scan_compacted"].append(float(lib.acb_last_kernel_ms()))
            kern["compact"].append(cm.value)
            kern["remap"].append(rm.value)
            runs["plain"]()
            kern["scan_plain"].append(float(lib.acb_last_kernel_ms()))
            kern["copy"].append(ev_time(runs["copy"]))
    finally:
        lib.acb_set_kernel_timing(0)
    kmed = {k: float(np.median(v)) for k, v in kern.items()}
    name, power = _card()
    med = {k: float(np.median(v)) for k, v in times.items()}
    res = {"card": name, "power_limit": power, "bytes": nbytes, "space_rate": a.rate, "reps": a.reps, "records": n_skip,
           "median_ms": med, "min_ms": {k: float(np.min(v)) for k, v in times.items()},
           "kernel_median_ms": kmed, "compact_over_copy": kmed["compact"] / kmed["copy"]}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "white_space.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
