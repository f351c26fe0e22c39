#!/usr/bin/env python3
"""Time the leftmost-longest replacement stage by stage on device-resident batches.

    python tools/time_replace.py [--reps 10] [--out DIR] [--kinds longest,first]

Workloads (pyahocorasick_b200.synth, C2's 10 k keys): C2 planted (1 M x 256 B), C4 (64 x 16 MiB), and C4's bytes as
one haystack of 1 GiB; each with three replacement tables: random lengths 0..24 (seeded), the identity (every key
mapped to itself) and delete-everything.  For each, with the batch resident in HBM:
  scan_ms        acb_scan_device (filter kernel) into a device buffer, the library's CUDA events around the launch
  select_ms      acb_leftmost_longest_device on that list, the sum of its stage times (acb_last_leftmost_ms)
  offsets_ms     acb_replace_device's offsets pass, write_ms its write pass (acb_last_replace_ms)
  d2d_ms         a device-to-device cudaMemcpyAsync of the output's byte count, CUDA events around it
  write_vs_d2d   write_ms / d2d_ms
  call_cuda_ms   a whole replace_batch from the CUDA tensor (host clock, ends in a synchronise)
  call_host_ms   a whole replace_batch from the host array (C2, C4) or (flat, offsets) pair (1 GiB)
Medians of `reps` runs after 2 warm-up runs.  Every output is checked once, piece by piece, against a numpy build from
find_leftmost_longest_batch's records.  The card's name, power limit and SM clocks are read in the same run.  Prints one
JSON line (also written to DIR/replace.json).  --kinds longest,first also times a leftmost-first replacer of the same
table (Automaton.replacer(leftmost_first=True)), its whole calls alternating with the leftmost-longest ones: each table
then has "first": {call_cuda_ms, call_host_ms} and "first_over_longest_cuda"."""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), [x.strip() for x in out.split(",")]))
    except Exception as e:                                      # the timings stand without it; say so
        return {"error": str(e)}


def _np_piece(flat, s, ln, rl, rs, rep):
    """the output of one piece of text (1-byte letters) whose chosen matches start at s (piece coordinates)"""
    import numpy as np
    cov = np.zeros(flat.size + 1, dtype=np.int64)
    np.add.at(cov, s, 1)
    np.add.at(cov, s + ln, -1)
    keep = np.cumsum(cov[:-1]) == 0
    units = keep.astype(np.int64)
    units[s] += rl
    pos = np.zeros(flat.size + 1, dtype=np.int64)
    np.cumsum(units, out=pos[1:])
    out = np.empty(int(pos[-1]), dtype=np.uint8)
    out[pos[:-1][keep]] = flat[keep]
    j = np.arange(int(rl.sum())) - np.repeat(np.cumsum(rl) - rl, rl)
    out[np.repeat(pos[s], rl) + j] = rep[np.repeat(rs, rl) + j]
    return out


def check(A, flat, in_off, rep, rep_off, out, out_off, pieces=64):
    """out / out_off against the numpy build from find_leftmost_longest_batch's records, in pieces cut at match starts"""
    import numpy as np
    m = A.find_leftmost_longest_batch((flat, in_off))
    kl = np.asarray(A.flat()["key_len"], dtype=np.int64)
    key = m.key_id.astype(np.int64)
    ln, rl = kl[key], rep_off[key + 1] - rep_off[key]
    s = in_off[m.hay_id.astype(np.int64)] + m.end_index.astype(np.int64) - ln + 1
    delta = np.zeros(len(in_off), dtype=np.int64)
    np.add.at(delta, m.hay_id.astype(np.int64) + 1, rl - ln)
    assert np.array_equal(out_off, in_off + np.cumsum(delta)), "output offsets"
    cuts = np.unique(np.concatenate([[0, flat.size], s[np.linspace(0, len(s) - 1, pieces).astype(np.int64)] if len(s) else []]))
    pos = 0
    for x0, x1 in zip(cuts[:-1].tolist(), cuts[1:].tolist()):
        i0, i1 = np.searchsorted(s, [x0, x1])
        piece = _np_piece(flat[x0:x1], s[i0:i1] - x0, ln[i0:i1], rl[i0:i1], rep_off[key[i0:i1]], rep)
        assert np.array_equal(out[pos:pos + piece.size], piece), ("bytes", x0)
        pos += piece.size
    assert pos == out.size


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    ap.add_argument("--kinds", default="longest", choices=["longest", "longest,first"])
    a = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to time")
    from pyahocorasick_b200 import _native as N
    from pyahocorasick_b200 import synth
    lib = N.lib()
    stream = torch.cuda.current_stream().cuda_stream
    c2, c4 = synth.make("C2"), synth.make("C4")
    A = synth.build_automaton(c2.keys)                         # C4 uses C2's key set
    tb = A._ensure_table(0)
    keys = [k for k in A._key_objs if k is not None]
    rng = np.random.default_rng(1)
    tables = {"random": {k: bytes(rng.integers(0x20, 0x7F, size=int(rng.integers(0, 25)), dtype=np.uint8)) for k in keys},
              "identity": {k: k for k in keys}, "delete": {k: b"" for k in keys}}
    work = {"C2": c2.haystacks, "C4": c4.haystacks, "1GiB": c4.haystacks.reshape(1, -1)}
    res = {"card": _card(), "reps": a.reps}
    med = lambda xs: float(np.median(xs))                      # noqa: E731
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for name, host in work.items():
        d = torch.from_numpy(host).cuda()
        n, stride = d.shape
        flat = host.reshape(-1)
        in_off = np.arange(n + 1, dtype=np.int64) * stride
        cnt = torch.zeros(1, dtype=torch.int64, device="cuda")
        cap = 1 << 24
        full = torch.empty((cap, 3), dtype=torch.int32, device="cuda")
        chosen = torch.empty((cap, 3), dtype=torch.int32, device="cuda")
        sel = torch.zeros(1, dtype=torch.int64, device="cuda")
        out_off = torch.empty(n + 1, dtype=torch.int64, device="cuda")
        total = torch.empty(1, dtype=torch.int64, device="cuda")
        res[name] = {}
        for tname, table in tables.items():
            R = A.replacer(table)
            r = R._replacer(tb, False, 0)
            rep, rep_off = R._tables[False]
            ms2, ms5 = (ctypes.c_float * 2)(), (ctypes.c_float * 5)()
            rows = {k: [] for k in ("scan_ms", "select_ms", "offsets_ms", "write_ms", "d2d_ms")}
            out = None
            for it in range(2 + a.reps):
                lib.acb_set_kernel_timing(1)
                cnt.zero_()
                N.check(lib.acb_scan_device(tb, d.data_ptr(), n * stride, None, n, stride, full.data_ptr(), cap, cnt.data_ptr(),
                                            stream, N.ALGO_FILTER))
                scan = lib.acb_last_kernel_ms()
                m = int(cnt.item())
                assert m <= cap
                sel.zero_()
                N.check(lib.acb_leftmost_longest_device(tb, full.data_ptr(), m, n, stride, chosen.data_ptr(), cap, sel.data_ptr(), stream))
                N.check(lib.acb_last_leftmost_ms(ms5, 5))
                select = sum(ms5)
                args = (r, tb, d.data_ptr(), n * stride, None, n, stride, chosen.data_ptr(), max(m, 1), sel.data_ptr(), out_off.data_ptr())
                if out is None:
                    N.check(lib.acb_replace_device(*args, None, 0, total.data_ptr(), stream))
                    out = torch.empty(max(int(total.item()), 16), dtype=torch.uint8, device="cuda")
                    dst = torch.empty_like(out)
                N.check(lib.acb_replace_device(*args, out.data_ptr(), out.numel(), total.data_ptr(), stream))
                N.check(lib.acb_last_replace_ms(ms2, 2))
                lib.acb_set_kernel_timing(0)
                nb = int(total.item())
                ev0.record()
                dst[:nb].copy_(out[:nb])
                ev1.record()
                ev1.synchronize()
                if it >= 2:
                    for k, v in zip(rows, (scan, select, ms2[0], ms2[1], ev0.elapsed_time(ev1))):
                        rows[k].append(v)
            row = {k: med(v) for k, v in rows.items()}
            row["write_vs_d2d"] = row["write_ms"] / row["d2d_ms"]
            row["out_bytes"] = nb
            row["records"] = {"full": m, "chosen": int(sel.item())}
            check(A, flat, in_off, rep, rep_off, out[:nb].cpu().numpy(), out_off.cpu().numpy())
            row["checked"] = True
            hostform = host if name != "1GiB" else (flat, np.array([0, flat.size], dtype=np.int64))
            Rs = {"longest": R}
            if a.kinds == "longest,first":
                Rs["first"] = A.replacer(table, leftmost_first=True)
            for key_, batch in (("call_cuda_ms", d), ("call_host_ms", hostform)):
                ts = {k: [] for k in Rs}
                for it in range(4):
                    for k, RR in Rs.items():
                        torch.cuda.synchronize()
                        t0 = time.perf_counter()
                        RR.replace_batch(batch)
                        torch.cuda.synchronize()
                        if it:
                            ts[k].append((time.perf_counter() - t0) * 1e3)
                row[key_] = med(ts["longest"])
                if "first" in Rs:
                    row.setdefault("first", {})[key_] = med(ts["first"])
            if "first" in Rs:
                row["first_over_longest_cuda"] = row["first"]["call_cuda_ms"] / row["call_cuda_ms"]
                del Rs
            res[name][tname] = row
            del R
            out = None
            torch.cuda.empty_cache()
        del d, full, chosen
        torch.cuda.empty_cache()
    for t in tables:
        res[f"1GiB_vs_C4_{t}"] = res["1GiB"][t]["write_ms"] / res["C4"][t]["write_ms"]
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "replace.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
