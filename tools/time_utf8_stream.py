#!/usr/bin/env python3
"""Time UTF-8 stream batches (stream_batch(encoding="utf-8")): the carry's stage and commit against a copy, and feeds
against the str feeds of the same decoded text.

    python tools/time_utf8_stream.py [--reps 7] [--out DIR]

The text: C2's keys (unicode flavour) and 1 M streams fed 256-byte chunks of C2's text made ASCII, with two U+2019
(3 bytes each) inside every chunk and a third one split across every chunk boundary (E2 80 | 99), so every stream holds
2 bytes back after every feed and every staged chunk decodes to 250 letters (~1.2 % of them U+2019).  Every feed after
the first is in that steady state.
  stage      acb_utf8_carry_stage_device + acb_utf8_carry_commit_device on the CUDA tensor of chunks against a
             device-to-device copy of it (torch copy_), CUDA events, alternated
  feeds      find_all, leftmost-longest and replacing feeds of the UTF-8 CUDA tensor [1 M, 256] against the str feeds of
             the same decoded letters as a UTF-32 CUDA tensor [1 M, 1000], host clock to a device synchronise,
             alternated; plus, from one UTF-8 feed with kernel timing on, its decode (both passes) and encode times
             (acb_last_utf8_ms).  Goal: UTF-8 feed <= str feed + decode + 1.5 copies (+ encode when replacing).
  host       find_all feeds from host memory: a list of bytes and (flat, offsets) against the list of the decoded str
             fed to the str batch, alternated
Medians of `reps` runs after 2 warm-up runs of every variant; every UTF-8 answer is checked once against the str one.
The card's name, power limit and SM clocks are read in the same run.  Prints one JSON line (also written to
DIR/utf8_stream.json)."""
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


def chunks(c2, np):
    """uint8 [n, 256]: C2's text made ASCII, two U+2019 inside each row, E2 80 at its end and 99 at its start"""
    rng = np.random.default_rng(21)
    rows = np.where(c2 >= 0x80, c2 & 0x7F, c2).astype(np.uint8)
    n = rows.shape[0]
    rows[:, 0] = 0x99
    rows[:, 254:] = [0xE2, 0x80]
    a = rng.integers(1, 125, size=n)                             # two quotes at random places of [1, 254)
    b = rng.integers(128, 251, size=n)
    for col in (a, b):
        for j, v in enumerate(b"\xe2\x80\x99"):
            rows[np.arange(n), col + j] = v
    return rows


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
    rows = chunks(c2.haystacks, np)
    n = rows.shape[0]
    d8 = torch.from_numpy(rows).cuda()
    strs = [(b"\xe2\x80" + r[:-2].tobytes()).decode() for r in rows]   # each staged chunk in the steady state
    letters = len(strs[0])
    text = np.frombuffer("".join(strs).encode("utf-32-le"), np.uint8)
    d32 = torch.from_numpy(text.reshape(n, 4 * letters).copy()).cuda()
    res["shape"] = {"streams": n, "chunk_bytes": rows.shape[1], "letters_per_chunk": letters}

    # the stage and commit against a copy of the chunk bytes
    c = ctypes.c_void_p()
    N.check(lib.acb_utf8_carry_new(0, n, ctypes.byref(c)))
    span = d8.numel() + 3 * n
    staged = torch.empty(span, dtype=torch.uint8, device="cuda")
    soffs = torch.empty(n + 1, dtype=torch.int64, device="cuda")
    dst = torch.empty_like(d8)
    e = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    stage_ms, copy_ms = [], []
    for r in range(2 + a.reps):
        s = torch.cuda.current_stream().cuda_stream
        e[0].record()
        N.check(lib.acb_utf8_carry_stage_device(c, d8.data_ptr(), d8.numel(), None, n, rows.shape[1], None, 0, staged.data_ptr(),
                                                span, soffs.data_ptr(), s))
        N.check(lib.acb_utf8_carry_commit_device(c, None, n, s))
        e[1].record()
        e[2].record()
        dst.copy_(d8)
        e[3].record()
        e[3].synchronize()
        if r >= 2:
            stage_ms.append(e[0].elapsed_time(e[1]))
            copy_ms.append(e[2].elapsed_time(e[3]))
    lib.acb_utf8_carry_free(c)
    res["stage"] = {"stage_commit_ms": med(stage_ms), "copy_ms": med(copy_ms), "over_copy": med(stage_ms) / med(copy_ms)}
    res["goal_stage_within_1_5x_copy"] = res["stage"]["over_copy"] <= 1.5
    del staged, soffs, dst
    copy = res["stage"]["copy_ms"]

    # device feeds: UTF-8 against the str feed of the same letters as UTF-32
    feeds = {}
    for name, make in (("find_all", lambda **kw: A.stream_batch(n, **kw)),
                       ("leftmost_longest", lambda **kw: A.stream_batch(n, leftmost_longest=True, **kw)),
                       ("replace", lambda **kw: R.stream_batch(n, **kw))):
        U, S = make(encoding="utf-8", errors="replace"), make()
        U.feed(d8)                                                 # the first feed: a stray 99 opens every stream
        U.reset()
        U.feed(d8[:, 254:].contiguous())                           # every stream now holds E2 80: the steady state
        got, want = U.feed(d8), S.feed(d32)
        if name == "replace":
            gf, go = got
            wf, wo = want
            assert gf.numel() > 0
            assert gf.cpu().numpy().tobytes().decode() == wf.cpu().numpy().tobytes().decode("utf-32-le")
        else:
            assert len(got) > 0 and all(np.array_equal(getattr(got, f), getattr(want, f)) for f in ("hay_id", "end_index", "key_id"))
        ms = (ctypes.c_float * 3)()
        lib.acb_set_kernel_timing(1)
        U.feed(d8)
        lib.acb_set_kernel_timing(0)
        N.check(lib.acb_last_utf8_ms(ms, 3))
        t = alternate({"str_utf32": lambda: S.feed(d32), "utf8": lambda: U.feed(d8)})
        t["decode_ms"], t["encode_ms"] = ms[0] + ms[1], (ms[2] if name == "replace" else 0.0)
        t["bound_ms"] = t["str_utf32"] + t["decode_ms"] + 1.5 * copy + t["encode_ms"]
        t["goal_met"] = t["utf8"] <= t["bound_ms"]
        feeds[name] = t
        del U, S
        torch.cuda.empty_cache()
    res["device_feeds"] = feeds

    # from host memory: find_all feeds
    as_bytes = [r.tobytes() for r in rows]
    offs = np.arange(n + 1, dtype=np.int64) * rows.shape[1]
    pair = (rows.reshape(-1), offs)
    U1, U2, S = (A.stream_batch(n, encoding="utf-8"), A.stream_batch(n, encoding="utf-8"), A.stream_batch(n))
    for U in (U1, U2):
        U.feed([b"\xe2\x80"] * n)
    got, want = U1.feed(as_bytes), S.feed(strs)
    assert len(got) > 0 and all(np.array_equal(getattr(got, f), getattr(want, f)) for f in ("hay_id", "end_index", "key_id"))
    res["host_find_all"] = alternate({"str": lambda: S.feed(strs), "utf8_list": lambda: U1.feed(as_bytes),
                                      "utf8_pair": lambda: U2.feed(pair)})
    h = res["host_find_all"]
    res["goal_host_utf8_faster"] = h["utf8_list"] < h["str"] and h["utf8_pair"] < h["str"]
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "utf8_stream.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
