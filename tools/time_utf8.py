#!/usr/bin/env python3
"""Time UTF-8 batches (encoding="utf-8"): the two decode passes against a copy, and whole calls against the same text
given as str or as UTF-32.

    python tools/time_utf8.py [--reps 7] [--out DIR]

  decode     acb_utf8_decode_device + acb_utf8_write_device at 4 bytes per letter (acb_last_utf8_ms) against a
             cudaMemcpyAsync device-to-device copy of the decoded buffer (torch copy_, CUDA events), alternated, on C2-shaped
             text (1 M x 256 bytes): "ascii" (C2's text), "curly" (C2's text with ~1 % of its letters replaced by U+2019,
             3 bytes each), "cjk" (85 random letters of U+4E00-U+9FFF and a space per row) and "invalid" (C2's text with
             ~1 % of its bytes 0xFF, errors="replace").  "ascii" is timed at 1 byte per letter too (its copy: the same
             bytes).
  host       whole calls, host clock to a device synchronise, from host memory on C2's keys (unicode flavour):
             find_all_batch and Replacer.replace_batch on the decoded list of str against the UTF-8 text as a list of
             bytes and as (flat, offsets), alternated, on "ascii" and "curly"
  device     find_all_batch on a UTF-32 CUDA tensor [n, 4 * letters] against the UTF-8 CUDA tensor [n, 256] of the same
             text, alternated, on "ascii" and "cjk" (rows of equal letter counts)
Medians of `reps` runs after 2 warm-up runs of every variant; every UTF-8 answer is checked once against the str or
UTF-32 one.  The card's name, power limit and SM clocks are read in the same run.  Prints one JSON line (also written
to DIR/utf8.json)."""
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


def texts(c2, np):
    """the four C2-shaped texts as uint8 [n, 256]"""
    rng = np.random.default_rng(8)
    ascii_ = np.where(c2 >= 0x80, c2 & 0x7F, c2).astype(np.uint8)
    n = ascii_.shape[0]
    curly = ascii_.copy()
    k = n * 256 // 100 // 3                                      # 3 bytes per quote: ~1 % of the letters
    rows, cols = rng.integers(0, n, size=k), rng.integers(0, 254, size=k) // 3 * 3
    for j, b in enumerate(b"\xe2\x80\x99"):
        curly[rows, cols + j] = b
    cp = rng.integers(0x4E00, 0xA000, size=(n, 85)).astype(np.uint32)
    cjk = np.empty((n, 256), dtype=np.uint8)
    cjk[:, 0:255:3] = 0xE0 | cp >> 12
    cjk[:, 1:255:3] = 0x80 | ((cp >> 6) & 0x3F)
    cjk[:, 2:255:3] = 0x80 | (cp & 0x3F)
    cjk[:, 255] = 0x20
    invalid = ascii_.copy()
    invalid.reshape(-1)[rng.integers(0, invalid.size, size=invalid.size // 100)] = 0xFF
    return {"ascii": ascii_, "curly": curly, "cjk": cjk, "invalid": invalid}


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

    c2 = synth.make("C2")
    keys = [k.decode("latin-1") for k in c2.keys]
    A = synth.build_automaton(keys, uni)
    R = A.replacer({k: k.upper() for k in keys})
    T = texts(c2.haystacks, np)

    # the decode passes against a copy of their output
    ms = (ctypes.c_float * 2)()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    decode = {}
    for name, narrow in (("ascii", False), ("curly", False), ("cjk", False), ("invalid", False), ("ascii", True)):
        d = torch.from_numpy(T[name]).cuda()
        errors = N.UTF8_REPLACE if name == "invalid" else N.UTF8_STRICT
        b = A._utf8_batch(d, errors, 0, narrow_ok=narrow)
        dst = torch.empty_like(b.data)
        dec_ms, copy_ms = [], []
        lib.acb_set_kernel_timing(1)
        for i in range(2 + a.reps):
            b = A._utf8_batch(d, errors, 0, narrow_ok=narrow)
            N.check(lib.acb_last_utf8_ms(ms, 2))
            e0.record()
            dst.copy_(b.data)
            e1.record()
            e1.synchronize()
            if i >= 2:
                dec_ms.append(ms[0] + ms[1])
                copy_ms.append(e0.elapsed_time(e1))
        lib.acb_set_kernel_timing(0)
        tag = f"{name}/{1 if b.narrow else 4}"
        decode[tag] = {"utf8_bytes": d.numel(), "letter_bytes": b.data.numel(), "decode_ms": med(dec_ms), "copy_ms": med(copy_ms)}
        decode[tag]["decode_over_copy"] = decode[tag]["decode_ms"] / decode[tag]["copy_ms"]
        del d, dst, b
    res["decode"] = decode
    res["goal_decode_within_1_5x_copy"] = all(v["decode_over_copy"] <= 1.5 for k, v in decode.items() if k.endswith("/4"))
    torch.cuda.empty_cache()

    # whole calls from host memory: the decoded list of str against the UTF-8 bytes
    host = {}
    for name in ("ascii", "curly"):
        rows = T[name]
        as_bytes = [r.tobytes() for r in rows]
        strs = [h.decode() for h in as_bytes]
        offs = np.arange(rows.shape[0] + 1, dtype=np.int64) * rows.shape[1]
        pair = (rows.reshape(-1), offs)
        m_s, m_b = A.find_all_batch(strs), A.find_all_batch(as_bytes, encoding="utf-8")
        assert len(m_s) > 0 and all(np.array_equal(getattr(m_s, f), getattr(m_b, f)) for f in ("hay_id", "end_index", "key_id"))
        assert R.replace_batch(as_bytes[:1000], encoding="utf-8") == [s.encode() for s in R.replace_batch(strs[:1000])]
        t = alternate({"find_all/str": lambda: A.find_all_batch(strs),
                       "find_all/utf8_list": lambda: A.find_all_batch(as_bytes, encoding="utf-8"),
                       "find_all/utf8_pair": lambda: A.find_all_batch(pair, encoding="utf-8"),
                       "replace/str": lambda: R.replace_batch(strs),
                       "replace/utf8_list": lambda: R.replace_batch(as_bytes, encoding="utf-8"),
                       "replace/utf8_pair": lambda: R.replace_batch(pair, encoding="utf-8")})
        host[name] = t
        del as_bytes, strs
    res["host_C2"] = host
    res["goal_host_utf8_faster_on_curly"] = all(host["curly"][f"{k}/utf8_list"] < host["curly"][f"{k}/str"] and
                                                host["curly"][f"{k}/utf8_pair"] < host["curly"][f"{k}/str"]
                                                for k in ("find_all", "replace"))

    # device-resident: UTF-32 against UTF-8 of the same text
    dev = {}
    for name in ("ascii", "cjk"):
        rows = T[name]
        d8 = torch.from_numpy(rows).cuda()
        text = [r.tobytes().decode() for r in rows[:1]]
        width = len(text[0])
        u32 = np.frombuffer(rows.tobytes().decode().encode("utf-32-le"), np.uint8).reshape(rows.shape[0], 4 * width)
        d32 = torch.from_numpy(u32.copy()).cuda()
        m32, m8 = A.find_all_batch(d32), A.find_all_batch(d8, encoding="utf-8")
        assert all(np.array_equal(getattr(m32, f), getattr(m8, f)) for f in ("hay_id", "end_index", "key_id"))
        dev[name] = alternate({"utf32": lambda: A.find_all_batch(d32), "utf8": lambda: A.find_all_batch(d8, encoding="utf-8")})
        dev[name]["matches"] = len(m8)
        del d8, d32, u32
        torch.cuda.empty_cache()
    res["device_C2"] = dev
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "utf8.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
