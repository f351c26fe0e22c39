#!/usr/bin/env python3
"""Time ASCII case-insensitive matching (ascii_case_insensitive=True) against case-sensitive calls.

    python tools/time_fold.py [--reps 5] [--out DIR]

Workloads (pyahocorasick_b200.synth): C2 planted (1 M x 256 B) and C4 (64 x 16 MiB, with C2's keys), every letter of
the text with its case flipped at random (seed 17).  Key sets: C2's 10 k keys ("keys"), and those plus every key's
swapcase() ("swapcase", 20 k keys in groups of two, so find_all expands every match).
  fold_ms / copy_ms   the fold kernel inside acb_scan_device (acb_last_fold_ms) and a cudaMemcpyAsync device-to-device
                      copy of the same bytes (torch copy_, CUDA events), alternated
  expand_ms           the alias expansion of the last device find_all (swapcase key set)
  calls_ms            whole calls, host clock to a device synchronise: find_all_batch, find_leftmost_longest_batch,
                      find_leftmost_first_batch and Replacer.replace_batch, each with ascii_case_insensitive False and
                      True, alternated, on the batch in HBM ("device") and in pinned host memory ("host"); on the device
                      also "find_all/folded", a case-sensitive find_all_batch of the folded text with the folded keys
                      (one per group), which finds what the folded call finds without folding anything
Medians of `reps` runs after 2 warm-up runs of every variant.  Each folded answer is checked once against the
case-sensitive one over folded text with folded keys.  The card's name, power limit and SM clocks are read in the same
run.  Prints one JSON line (also written to DIR/fold.json)."""
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


def _flip(hay, seed=17):
    import numpy as np
    rng = np.random.default_rng(seed)
    out = hay.copy()
    low = out | 0x20
    out[rng.integers(0, 2, size=out.shape).astype(bool) & (low >= 0x61) & (low <= 0x7A)] ^= 0x20
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to time")
    from pyahocorasick_b200 import _native as N
    from pyahocorasick_b200 import synth
    lib = N.lib()
    med = lambda xs: float(np.median(xs))                      # noqa: E731
    c2, c4 = synth.make("C2"), synth.make("C4")
    have = set(c2.keys)
    key_sets = {"keys": list(c2.keys), "swapcase": list(c2.keys) + [k.swapcase() for k in c2.keys if k.swapcase() not in have]}
    res = {"card": _card(), "reps": a.reps}

    def alternate(fns):
        """{name: median ms} of fns run in turn, host clock to a device synchronise"""
        out = {k: [] for k in fns}
        for r in range(2 + a.reps):
            for k, fn in fns.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn()
                torch.cuda.synchronize()
                if r >= 2:
                    out[k].append((time.perf_counter() - t0) * 1e3)
        return {k: med(v) for k, v in out.items()}

    for name, w in (("C2", c2), ("C4", c4)):
        host = _flip(w.haystacks)
        pinned = torch.empty(host.shape, dtype=torch.uint8).pin_memory()
        pinned.numpy()[:] = host
        hp = pinned.numpy()
        d = pinned.cuda()
        n, stride = d.shape
        for ks, keys in key_sets.items():
            if name == "C4" and ks == "swapcase":
                continue
            A = synth.build_automaton(keys)
            R = A.replacer({k: k.upper() for k in keys})
            # the check: the case-sensitive answers over folded text, with the folded keys in order of first appearance
            size = {}
            for k in keys:
                size[k.lower()] = size.get(k.lower(), 0) + 1
            F = synth.build_automaton(list(size))
            weight = np.array(list(size.values()), dtype=np.int64)
            folded = torch.from_numpy(host).cuda()
            low = folded | 0x20
            upper = (low >= 0x61) & (low <= 0x7A)
            folded[upper] = low[upper]
            got = A.find_leftmost_first_batch(d, ascii_case_insensitive=True)
            want = F.find_leftmost_first_batch(folded)
            assert np.array_equal(got.hay_id, want.hay_id) and np.array_equal(got.end_index, want.end_index), (name, ks)
            m = A.find_all_batch(d, ascii_case_insensitive=True)
            assert len(m) == int(weight[F.find_all_batch(folded).key_id].sum()), (name, ks)
            del low, upper
            r = {"records": len(m)}
            # the fold kernel against a copy of the same bytes
            tb = A._table_for(0, False, True)
            cap = max(len(m), 1) + 1024
            rec = torch.empty((cap, 3), dtype=torch.int32, device="cuda")
            cnt = torch.zeros(1, dtype=torch.int64, device="cuda")
            dst = torch.empty_like(d)
            stream = torch.cuda.current_stream().cuda_stream
            ms = (ctypes.c_float * 2)()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            fold_ms, copy_ms = [], []
            lib.acb_set_kernel_timing(1)
            for i in range(2 + a.reps):
                cnt.zero_()
                N.check(lib.acb_scan_device(tb, d.data_ptr(), n * stride, None, n, stride, rec.data_ptr(), cap, cnt.data_ptr(),
                                            stream, N.ALGO_FILTER))
                N.check(lib.acb_last_fold_ms(ms, 2))
                e0.record()
                dst.copy_(d)
                e1.record()
                e1.synchronize()
                if i >= 2:
                    fold_ms.append(ms[0])
                    copy_ms.append(e0.elapsed_time(e1))
            A.find_all_batch(d, ascii_case_insensitive=True)
            N.check(lib.acb_last_fold_ms(ms, 2))
            lib.acb_set_kernel_timing(0)
            r.update(fold_ms=med(fold_ms), copy_ms=med(copy_ms), expand_ms=float(ms[1]))
            r["fold_over_copy"] = r["fold_ms"] / r["copy_ms"]
            del dst, rec
            for where, b in (("device", d), ("host", hp)):
                fns = {}
                for fold in (False, True):
                    tag = "ci" if fold else "cs"
                    fns[f"find_all/{tag}"] = lambda f=fold: A.find_all_batch(b, ascii_case_insensitive=f)
                    fns[f"longest/{tag}"] = lambda f=fold: A.find_leftmost_longest_batch(b, ascii_case_insensitive=f)
                    fns[f"first/{tag}"] = lambda f=fold: A.find_leftmost_first_batch(b, ascii_case_insensitive=f)
                    fns[f"replace/{tag}"] = lambda f=fold: R.replace_batch(b, ascii_case_insensitive=f)
                if where == "device":                           # the same search without the fold: folded text, folded keys
                    fns["find_all/folded"] = lambda: F.find_all_batch(folded)
                t = alternate(fns)
                for k in ("find_all", "longest", "first", "replace"):
                    t[f"{k}/ratio"] = t[f"{k}/ci"] / t[f"{k}/cs"]
                if where == "device":
                    t["find_all/ci_over_folded"] = t["find_all/ci"] / t["find_all/folded"]
                r[where] = t
            r["device_find_all_goal_ms"] = r["device"]["find_all/cs"] + 1.25 * r["copy_ms"]
            res[f"{name}/{ks}"] = r
            del A, R, F, folded
            torch.cuda.empty_cache()
        del d, pinned
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "fold.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
