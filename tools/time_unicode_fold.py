#!/usr/bin/env python3
"""Time Unicode case-insensitive matching (case_insensitive=True): its fold kernel against a copy, and whole calls
against ascii_case_insensitive=True.

    python tools/time_unicode_fold.py [--reps 7] [--out DIR]

  fold            the fold kernel inside acb_scan_device on the Unicode-folded table (acb_last_fold_ms) against a
                  cudaMemcpyAsync device-to-device copy of the same bytes (torch copy_, CUDA events), alternated; 64 M
                  letters each.  4-byte letters: "ascii" (C2's text, case flipped at random), "greek_cyrillic" (Greek and
                  Cyrillic capitals and smalls at random), "every_changed" (every code point the fold changes, at random:
                  all table blocks); 1-byte letters: "latin1" (A-Z, a-z and U+00C0-U+00FE at random)
  calls           C2's keys and text (1 M x 256 letters, ASCII, case flipped at random) in the unicode flavour at 4 bytes
                  per letter: whole calls, host clock to a device synchronise, of find_all_batch,
                  find_leftmost_longest_batch and Replacer.replace_batch with case_insensitive against
                  ascii_case_insensitive, alternated, on the batch in HBM ("device") and in pinned host memory ("host")
Medians of `reps` runs after 2 warm-up runs of every variant.  Each case_insensitive answer is checked once against
the ascii_case_insensitive one.  The card's name, power limit and SM clocks are read in the same run.  Prints one JSON
line (also written to DIR/unicode_fold.json)."""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.time_fold import _flip  # noqa: E402
from tools.time_leftmost import _card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to time")
    import pyahocorasick_b200 as pkg
    from pyahocorasick_b200 import _native as N
    from pyahocorasick_b200 import synth
    from pyahocorasick_b200.automaton import _FOLD_UNICODE, _unicode_fold_map
    lib = N.lib()
    uni = pkg.flavour("unicode")
    med = lambda xs: float(np.median(xs))                      # noqa: E731
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

    # the fold kernel against a copy
    c2 = synth.make("C2")
    n = 64 << 20
    rng = np.random.default_rng(5)
    frm = _unicode_fold_map()[0]
    greek_cyrillic = np.concatenate([np.arange(0x391, 0x3AA), np.arange(0x3B1, 0x3CA), np.arange(0x410, 0x450)])
    latin1 = np.concatenate([np.arange(0x41, 0x5B), np.arange(0x61, 0x7B), np.arange(0xC0, 0xFF)])
    texts = {"ascii": _flip(c2.haystacks.reshape(-1)[:n]).astype("<u4"),
             "greek_cyrillic": rng.choice(greek_cyrillic, size=n).astype("<u4"),
             "every_changed": rng.choice(frm, size=n).astype("<u4"),
             "latin1": rng.choice(latin1, size=n).astype(np.uint8)}
    A = synth.build_automaton(["☃☃", "\xd7\xf7\xd7\xf7"], uni)
    ms = (ctypes.c_float * 2)()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    stream = torch.cuda.current_stream().cuda_stream
    rec = torch.empty((1 << 16, 3), dtype=torch.int32, device="cuda")
    cnt = torch.zeros(1, dtype=torch.int64, device="cuda")
    fold = {}
    for name, t in texts.items():
        d = torch.from_numpy(t.view(np.uint8)).cuda()
        dst = torch.empty_like(d)
        tb = A._table_for(0, t.dtype == np.uint8, _FOLD_UNICODE)
        fold_ms, copy_ms = [], []
        lib.acb_set_kernel_timing(1)
        for i in range(2 + a.reps):
            cnt.zero_()
            N.check(lib.acb_scan_device(tb, d.data_ptr(), d.numel(), None, 1, d.numel(), rec.data_ptr(), rec.shape[0],
                                        cnt.data_ptr(), stream, N.ALGO_FILTER))
            N.check(lib.acb_last_fold_ms(ms, 1))
            e0.record()
            dst.copy_(d)
            e1.record()
            e1.synchronize()
            if i >= 2:
                fold_ms.append(ms[0])
                copy_ms.append(e0.elapsed_time(e1))
        lib.acb_set_kernel_timing(0)
        fold[name] = {"letter_bytes": t.dtype.itemsize, "bytes": d.numel(), "fold_ms": med(fold_ms), "copy_ms": med(copy_ms)}
        fold[name]["fold_over_copy"] = fold[name]["fold_ms"] / fold[name]["copy_ms"]
        del d, dst
    res["fold"] = fold
    del texts
    torch.cuda.empty_cache()

    # whole calls: case_insensitive against ascii_case_insensitive on ASCII keys and text
    keys = [k.decode("latin-1") for k in c2.keys]
    A = synth.build_automaton(keys, uni)
    R = A.replacer({k: k.upper() for k in keys})
    wide = _flip(c2.haystacks).astype("<u4").view(np.uint8)
    pinned = torch.empty(wide.shape, dtype=torch.uint8).pin_memory()
    pinned.numpy()[:] = wide
    del wide
    hp = pinned.numpy()
    d = pinned.cuda()
    for ci, ai in ((A.find_all_batch(d, case_insensitive=True), A.find_all_batch(d, ascii_case_insensitive=True)),
                   (A.find_leftmost_longest_batch(hp, case_insensitive=True), A.find_leftmost_longest_batch(hp, ascii_case_insensitive=True))):
        assert len(ci) > 0 and all(np.array_equal(getattr(ci, f), getattr(ai, f)) for f in ("hay_id", "end_index", "key_id"))
    calls = {}
    for where, b in (("device", d), ("host", hp)):
        fns = {}
        for tag, kw in (("ascii", {"ascii_case_insensitive": True}), ("unicode", {"case_insensitive": True})):
            fns[f"find_all/{tag}"] = lambda kw=kw: A.find_all_batch(b, **kw)
            fns[f"longest/{tag}"] = lambda kw=kw: A.find_leftmost_longest_batch(b, **kw)
            fns[f"replace/{tag}"] = lambda kw=kw: R.replace_batch(b, **kw)
        t = alternate(fns)
        for k in ("find_all", "longest", "replace"):
            t[f"{k}/ratio"] = t[f"{k}/unicode"] / t[f"{k}/ascii"]
        calls[where] = t
    res["calls_C2"] = calls
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "unicode_fold.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
