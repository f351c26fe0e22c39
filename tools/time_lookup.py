#!/usr/bin/env python3
"""Time the lookup stage of the reference's published benchmark, per key and as one batch.

    python tools/time_lookup.py [--words 1000000] [--flavour bytes|unicode|both] [--reps 20] [--out DIR]

The workload is the lookup stage of the reference's etc/benchmarks/benchmark.py:79-86 with the word generator of
tools/published_benchmark.py: N random words of 3..32 characters over [a-zA-Z0-9], each stored with itself as value,
then N lookups of those words and N of words that are not keys (2 N in all, one list).  For each flavour it reports:
  reference_loop_s   the reference extension's get(w, None) loop (oracle/_ref, when it is built)
  per_key_loop_s     the drop-in's get(w, None) loop (one ctypes call into the host trie per key)
  get_batch_s        get_batch(list, None), host clock around the call, table already uploaded (median of 5), split
                     into the list's conversion to one buffer, acb_lookup_host (upload, kernel, copy back) and the
                     mapping of key ids to values
  upload_s           acb_table_upload of the automaton on its own
  kernel_ms          acb_lookup_device on device-resident keys and offsets: CUDA events around the launch (the
                     library's kernel timing), median of `reps` launches after 3 warm-up launches, and lookups/s
All paths must return the same answers.  The card's name and power limit are read in the same run.  Prints one JSON
line (also written to DIR/lookup.json)."""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import random
import string
import subprocess
import sys
import time

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


def words_and_misses(n: int):
    """tools/published_benchmark.py's words (same generator and seed), then n more words that are not among them"""
    rng = random.Random(0)
    chars = string.ascii_letters + string.digits
    seen = set()
    while len(seen) < n:
        seen.add("".join(rng.choice(chars) for _ in range(rng.randint(3, 32))))
    miss = set()
    while len(miss) < n:
        w = "".join(rng.choice(chars) for _ in range(rng.randint(3, 32)))
        if w not in seen:
            miss.add(w)
    return list(seen), list(miss)


def _clock(fn):
    t0 = time.perf_counter()
    r = fn()
    return time.perf_counter() - t0, r


def run(flavour: str, words, miss, reps: int) -> dict:
    import numpy as np
    import torch
    import pyahocorasick_b200 as pkg
    from pyahocorasick_b200 import _native as N
    conv = (lambda s: s.encode()) if flavour == "bytes" else (lambda s: s)
    keys = [conv(w) for w in words]
    q = keys + [conv(w) for w in miss]
    A = pkg.flavour(flavour).Automaton()
    for k in keys:
        A.add_word(k, k)
    A.make_automaton()
    out = {"keys": len(keys), "lookups": len(q)}

    out["per_key_loop_s"], want = _clock(lambda: [A.get(k, None) for k in q])
    import oracle
    if oracle.ref_available(flavour):
        R = oracle.ref_module(flavour).Automaton()
        for k in keys:
            R.add_word(k, k)
        R.make_automaton()
        out["reference_loop_s"], ref = _clock(lambda: [R.get(k, None) for k in q])
        assert ref == want, "the reference and the drop-in's get() disagree"
        del R

    A._drop_table()
    out["upload_s"], _ = _clock(lambda: A._ensure_table(0))
    got = A.get_batch(q, None)                                  # warm-up
    assert got == want, "get_batch differs from the get() loop"
    t = []
    for _ in range(5):
        dt, got = _clock(lambda: A.get_batch(q, None))
        assert got == want
        t.append(dt)
    out["get_batch_s"] = float(np.median(t))
    conv_s, native_s = [], []
    for _ in range(5):                                          # where get_batch's time goes
        dt, batch = _clock(lambda: A._batch_input(q, narrow_ok=False, required=False))
        conv_s.append(dt)
        _, flat, offs, n, stride, _ = batch
        dt, _ = _clock(lambda: A._lookup_host(flat, offs, n, stride, 0))
        native_s.append(dt)
    out["get_batch_split_s"] = {"list_to_buffer": float(np.median(conv_s)), "acb_lookup_host": float(np.median(native_s)),
                                "ids_to_values": out["get_batch_s"] - float(np.median(conv_s)) - float(np.median(native_s))}
    out["query_bytes"] = int(flat.size)

    # the kernel alone, on device-resident keys and offsets
    lib = N.lib()
    tb = A._ensure_table(0)
    d_keys = torch.from_numpy(flat.copy()).cuda()                # a writable copy: torch does not wrap read-only arrays
    d_offs = torch.from_numpy(offs).cuda()
    kid = torch.empty(n, dtype=torch.int32, device="cuda")
    pre = torch.empty(n, dtype=torch.int32, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    torch.cuda.synchronize()
    lib.acb_set_kernel_timing(1)
    ms = []
    try:
        for i in range(3 + reps):
            N.check(lib.acb_lookup_device(tb, d_keys.data_ptr(), int(flat.size), d_offs.data_ptr(), n, 0,
                                          kid.data_ptr(), pre.data_ptr(), stream))
            if i >= 3:
                ms.append(float(lib.acb_last_kernel_ms()))
    finally:
        lib.acb_set_kernel_timing(0)
    host_kid, _ = A._lookup_host(flat, offs, n, stride, 0)
    assert (kid.cpu().numpy() == host_kid).all()
    out["kernel_ms"] = {"median": float(np.median(ms)), "min": float(np.min(ms)), "max": float(np.max(ms)), "launches": reps}
    out["kernel_lookups_per_s"] = n / (float(np.median(ms)) * 1e-3)
    fv = N.FlatView()
    N.check(lib.acb_trie_flat_view(A._trie, ctypes.byref(fv)))
    out["table"] = {"states": fv.n_states, "classes": fv.n_classes, "goto_bytes": fv.n_states * fv.n_classes * 4}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--words", type=int, default=1_000_000)
    ap.add_argument("--flavour", default="both", choices=["bytes", "unicode", "both"])
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to time")
    if a.reps < 20:
        raise SystemExit("--reps must be at least 20")
    words, miss = words_and_misses(a.words)
    res = {"workload": f"{a.words} keys of 3..32 chars over [a-zA-Z0-9]; {a.words} present + {a.words} absent lookups",
           "published_lookup_2n_s_xeon_e3_1505m_v6": 1.307}
    for fl in (["bytes", "unicode"] if a.flavour == "both" else [a.flavour]):
        res[fl] = run(fl, words, miss, a.reps)
    res["card"], res["power_limit"] = _card()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "lookup.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
