#!/usr/bin/env python3
"""Case-folded stream feeds (DESIGN 4.18) against the plain feeds, batch resident in HBM.

    python tools/time_stream_fold.py [--config C2 C4] [--steps 30] [--warmup 3] [--no-swapcase]

As tools/time_stream_words.py does, each configuration's batch is fed as the next chunk of every stream (C2: 1 M streams
x 256 B; C4: 64 streams x 16 MiB), warmup + steps times in a row.  The text is the configuration's with every ASCII
letter's case flipped at random.  Each feed kind (find_all, leftmost-longest, leftmost-first, replacing, find_all with
whole words) runs in three variants, alternated within every step, each timed with CUDA events around the whole call:
  (a) the plain feed on the original text with the original keys;
  (b) the folded feed (acb_streams_new_folded) on the case-flipped text;
  (c) the plain feed on text folded beforehand, with the keys folded beforehand: the same matches, nothing to fold.
A device-to-device copy of the bytes a feed folds (the chunks for find_all, held + chunk for the others) is timed in the
same steps (both copies warmed up, their order alternated, the median of three in a row per step); the goal of a folded feed is (c) + 1.25 such copies.  A second pass with the library's kernel timing on
gives the fold and alias-expansion times of the folded feeds (acb_last_fold_ms).  On C2, one more pass adds every key's
swapcase() to the key set (groups of two), for the expansion's share of the find_all feeds.  Prints one JSON line per
configuration and pass, with the card's name, power limit and SM clocks read in the same run."""
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


KINDS = ("find_all", "leftmost", "first", "replace", "w_find_all")
WORDS = b"abcdefghijklmnopqrstuvwxyz"


def flip(hay, rng):
    out = hay.copy()
    f = rng.integers(0, 2, size=out.shape).astype(bool) & (((out | 0x20) >= 0x61) & ((out | 0x20) <= 0x7A))
    out[f] ^= 0x20
    return out


def lower(x):
    return np.where((x >= 0x41) & (x <= 0x5A), x + 0x20, x).astype(np.uint8)


class Variant:
    """one automaton's table, text and stream batches of every kind"""

    def __init__(self, keys, text, fold, n, stride):
        self.A = synth.build_automaton(keys)
        self.L = N.lib()
        self.A._ensure_table(0)
        self.tb = self.A._table_for(0, False, True) if fold else self.A._ensure_table(0)
        self.fold = fold
        self.d = torch.from_numpy(text).cuda()
        self.n, self.stride, self.total = n, stride, int(text.size)
        rng = np.random.default_rng(1)
        ks = [k for k in self.A._key_objs if k is not None]
        R = self.A.replacer({k: bytes(rng.integers(0x41, 0x5B, size=int(rng.integers(0, 20)), dtype=np.uint8)) for k in ks})
        self.R = R
        self.r = {N.SELECT_LONGEST: R._replacer(self.tb, False, 0)}
        bits, n_bits = _word_bits(("bytes", WORDS), 1)
        self.h = {}
        L = self.L
        for kind in KINDS:
            ss = ctypes.c_void_p()
            sel = N.SELECT_FIRST if kind == "first" else N.SELECT_LONGEST
            if fold:
                b = (N.ptr(bits), n_bits) if kind == "w_find_all" else (None, -1)
                N.check(L.acb_streams_new_folded(self.tb, n, int(kind in ("leftmost", "first", "replace")), sel, *b, ctypes.byref(ss)))
            elif kind == "find_all":
                N.check(L.acb_streams_new(self.tb, n, 0, ctypes.byref(ss)))
            elif kind == "w_find_all":
                N.check(L.acb_streams_new_words(self.tb, n, 0, N.ptr(bits), n_bits, ctypes.byref(ss)))
            else:
                N.check(L.acb_streams_new_leftmost_kind(self.tb, n, sel, None, -1, ctypes.byref(ss)))
            self.h[kind] = ss

    def feed(self, kind, io):
        L, ss, d, n, stride, total = self.L, self.h[kind], self.d, self.n, self.stride, self.total
        stream, algo = torch.cuda.current_stream().cuda_stream, N.ALGOS["auto"]
        if kind == "find_all":
            N.check(L.acb_streams_feed_device(ss, self.tb, d.data_ptr(), total, None, n, stride, None, io["out"].data_ptr(), io["cap"],
                                              io["cnt"].data_ptr(), stream, algo))
        elif kind == "w_find_all":
            N.check(L.acb_streams_feed_words_device(ss, self.tb, d.data_ptr(), total, None, n, stride, None, 0, io["out"].data_ptr(),
                                                    io["cap"], io["cnt"].data_ptr(), stream, algo))
        elif kind in ("leftmost", "first"):
            N.check(L.acb_streams_feed_leftmost_device(ss, self.tb, d.data_ptr(), total, None, n, stride, None, 0, io["out"].data_ptr(),
                                                       io["cap"], io["cnt"].data_ptr(), stream, algo))
        else:
            N.check(L.acb_streams_replace_device(ss, self.r[N.SELECT_LONGEST], self.tb, d.data_ptr(), total, None, n, stride, None, 0,
                                                 io["r_off"].data_ptr(), io["r_out"].data_ptr(), io["out_cap"], io["r_tot"].data_ptr(),
                                                 stream, algo))
        return int(io["r_tot"].item()) if kind == "replace" else int(io["cnt"].item())

    def free(self):
        for ss in self.h.values():
            self.L.acb_streams_free(ss)


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def run(config, steps, warmup, swapcase, kinds):
    w = synth.make(config, scale=1.0)
    n, stride = w.haystacks.shape
    keys = list(w.keys)
    if swapcase:
        have = set(keys)
        keys += [k.swapcase() for k in w.keys if k.swapcase() not in have]
    folded_keys = sorted({bytes(lower(np.frombuffer(k, np.uint8))) for k in keys})
    text = flip(w.haystacks, np.random.default_rng(2))
    variants = {"a": Variant(list(w.keys), w.haystacks, False, n, stride), "b": Variant(keys, text, True, n, stride),
                "c": Variant(folded_keys, lower(text), False, n, stride)}
    total = int(text.size)
    cap = max(8 * n, 1 << 25)
    io = {"out": torch.empty((cap, 3), dtype=torch.int32, device="cuda"), "cap": cap,
          "cnt": torch.zeros(1, dtype=torch.int64, device="cuda"), "out_cap": total * 5 // 4 + (1 << 22)}
    io.update(r_out=torch.empty(io["out_cap"], dtype=torch.uint8, device="cuda"), r_off=torch.empty(n + 1, dtype=torch.int64, device="cuda"),
              r_tot=torch.zeros(1, dtype=torch.int64, device="cuda"))
    T = int(variants["a"].A.get_stats()["longest_word"]) - 1
    staged = total + n * T                                       # at most: every stream holds T letters back
    src = torch.empty(staged, dtype=torch.uint8, device="cuda")
    dst = torch.empty_like(src)
    copies = {"chunks": lambda: dst[:total].copy_(src[:total]), "staged": lambda: dst.copy_(src)}
    for _ in range(warmup):
        for c in copies.values():
            c()
        for k in kinds:
            for v in variants.values():
                v.feed(k, io)
    torch.cuda.synchronize()
    ms = {(k, v): [] for k in kinds for v in variants}
    counts = {}
    copy_ms = {"chunks": [], "staged": []}
    for step in range(steps):
        for c in (("chunks", "staged") if step % 2 else ("staged", "chunks")):      # alternated, 3 in a row each
            copy_ms[c].append(float(np.median([timed(copies[c]) for _ in range(3)])))
        for k in kinds:
            for name, v in variants.items():
                ms[(k, name)].append(timed(lambda: counts.__setitem__((k, name), v.feed(k, io))))
    assert all(c <= cap for (k, _), c in counts.items() if k != "replace")
    L = N.lib()
    L.acb_set_kernel_timing(1)
    fold_split = {k: [] for k in kinds}
    f = (ctypes.c_float * 2)()
    for _ in range(min(steps, 10)):
        for k in kinds:
            fm = timed(lambda: variants["b"].feed(k, io))
            N.check(L.acb_last_fold_ms(f, 2))
            fold_split[k].append((f[0], f[1], fm))
    L.acb_set_kernel_timing(0)
    for v in variants.values():
        v.free()
    copy = {x: med(v) for x, v in copy_ms.items()}
    res = {"config": config, "swapcase_keys": swapcase, "n_streams": n, "chunk_bytes": stride, "tail_letters": T,
           "copy_ms": copy}
    for k in kinds:
        a, b, c = (med(ms[(k, x)]) for x in "abc")
        bytes_folded = copy["chunks"] if k == "find_all" else copy["staged"]
        res[k] = {"a_plain_ms": a, "b_folded_ms": b, "c_prefolded_ms": c, "b_over_c": round(b / c, 3), "b_over_a": round(b / a, 3),
                  "goal_ms": round(c + 1.25 * bytes_folded, 4), "goal_met": b <= c + 1.25 * bytes_folded,
                  "fold_ms": med([x[0] for x in fold_split[k]]), "expand_ms": med([x[1] for x in fold_split[k]]),
                  "expand_share": round(med([x[1] for x in fold_split[k]]) / max(med([x[2] for x in fold_split[k]]), 1e-9), 4),
                  "records_b": counts[(k, "b")], "records_c": counts[(k, "c")]}
    return {**res, **card()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", nargs="+", default=["C2", "C4"])
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--no-swapcase", action="store_true", help="skip the C2 pass with every key's swapcase() added")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_stream_fold.py needs a CUDA device")
    for c in args.config:
        print(json.dumps(run(c, args.steps, args.warmup, False, KINDS)), flush=True)
        torch.cuda.empty_cache()
    if not args.no_swapcase and "C2" in args.config:
        print(json.dumps(run("C2", args.steps, args.warmup, True, ("find_all", "w_find_all"))), flush=True)


if __name__ == "__main__":
    main()
