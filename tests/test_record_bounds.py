"""The record buffer's bounds and the record sort, against the oracle and a plain numpy restatement.

Record capacity.  Every kernel stores a record through `g = atomicAdd(count)` and `if (g < cap)`: the warp staging of the
stream kernel (emit, flush_stage), the pair kernel's emit_direct and batched resolve, the DFA and the iter_long kernel, and in a stream-batch feed the
seam kernel and the iter_long kernel with per-stream start states.
The callers' retry depends on two things: the count is exact when the buffer overflows, and nothing is written at or
past `cap`.  Each kernel here writes into an int32[cap + GUARD, 3] torch buffer filled with -1 that is passed with
capacity `cap`, so an overrun lands in the guard rows of the same allocation.  acb_scan_host is checked the same way on
its monolithic and its pipelined route: ACB_EOVERFLOW with the exact count, cap == n, and a caller buffer with guard rows.

Record sort.  acb_sort_matches_device packs hay_id | end_index | max_len - len into bits_for(n_hay - 1) +
bits_for(max_letters) + bits_for(max_len) bits of one radix key and returns ACB_ERANGE above 64.  Synthetic records put
every field at a power-of-two boundary and are compared with a stable numpy lexsort; the callers' fallbacks (std::sort in
acb_scan_host, np.lexsort in the device-tensor entry) are reached through a key set with one very long key and through
a wrapped library call.
"""
import ctypes

import numpy as np
import pytest

import oracle
import pyahocorasick_b200 as ac
from pyahocorasick_b200 import _native as N
from pyahocorasick_b200 import synth
from batch_cases import triples
from kernel_cells import SLICE, Cell, _big_batch, _build, _check_shape, _dense, _keys, _seed, tile_bytes

GUARD = 64
MiB = 1 << 20


def bits_for(v):
    """the library's field width (acb_device.cu): bits of v, at least 1"""
    b = 1
    while b < 64 and v >> b:
        b += 1
    return b


def sort_bits(n_hay, max_letters, max_len):
    return bits_for(max(n_hay - 1, 1)) + bits_for(max(max_letters, 1)) + bits_for(max_len)


def _oracle(keys):
    O = oracle.OracleAutomaton()
    for i, k in enumerate(keys):
        O.add_word(k, i)
    O.make_automaton()
    return O


def _tuples(a):
    return [tuple(r) for r in np.asarray(a).tolist()]


# ------------------------------------------------------------------ the kernels' write sites
PAIR_KEYS = [b"abab", b"baba", b"ababab", b"abcd"]          # "abab" / "ababab": a MULTI anchor; "abcd": UNIQUE


def _pair_text():
    t = np.frombuffer(b"ab" * 3000 + b"abcd" * 200 + b"ab" * 1000 + b"xabcdx" * 50, dtype=np.uint8).copy()
    off = np.array([0, 1000, 1001, 1001, 6000, t.size], dtype=np.int64)
    return t, off


def _case(name, monkeypatch):
    """(automaton, algo, text, offsets, the oracle's records as a list)"""
    if name == "pair_multi":                                       # one MULTI anchor: every record goes through emit_direct
        keys = [b"abab", b"ababab", b"abababab"]
        A = synth.build_automaton(keys)
        f = A.flat()
        assert f["filter_flags"] & 2 and (f["anchors"][f["anchors"][:, 0] != 0][:, 1] == 0xFFFFFFFF).all()
        t = np.frombuffer(b"ab" * 4000, dtype=np.uint8).copy()
        off = np.array([0, 3001, 3001, t.size], dtype=np.int64)
        return A, N.ALGO_FILTER, t, off, _tuples(_oracle(keys).scan_batch_bytes(t, off))
    if name in ("pair", "dfa", "long"):
        A = synth.build_automaton(PAIR_KEYS)
        assert A.filter_shape()["filter_flags"] & 2                # the pair kernel
        t, off = _pair_text()
        O = _oracle(PAIR_KEYS)
        if name == "long":
            want = O.iter_long_batch_letters(t, off)
        else:
            want = _tuples(O.scan_batch_bytes(t, off))
        return A, {"pair": N.ALGO_FILTER, "dfa": N.ALGO_DFA, "long": N.ALGO_LONG}[name], t, off, want
    cell = Cell(1, 3, 1) if name == "narrow" else Cell(1, 4, 1)
    keys = _keys(cell, np.random.Generator(np.random.PCG64(_seed(cell))))
    A = _build(cell, keys, monkeypatch)
    fs = _check_shape(A, cell)
    assert fs["filter_flags"] == (0 if name == "narrow" else 1)   # acb_stream_kernel, narrow / wide mode
    t = _dense(cell, tile_bytes(cell) + 3 * SLICE).astype(np.uint8)            # every probe a hit: the 64-record staging spills
    off = np.array([0, 7, 7, t.size // 2, t.size], dtype=np.int64)
    O = _oracle([bytes(k) for k in keys])
    return A, N.ALGO_FILTER, t, off, _tuples(O.scan_batch_bytes(t, off))


def _feed_case(name):
    """Stream-batch feeds through the C ABI (acb_streams_feed_device), after a first feed that leaves every stream
    with a tail or inside a key.  seam: every key has 6 letters or more and the second chunks have 4, so every record is
    written by the seam kernel; long_states: the iter_long kernel with per-stream start states.  Returns
    (automaton, algo, first chunks, (second chunks, offsets), the second feed's records: (chunk, end in it, key))."""
    rng = np.random.Generator(np.random.PCG64(606))
    ab = np.frombuffer(b"ab", dtype=np.uint8)
    if name == "seam":
        keys = [bytes(b"ab"[(i >> j) & 1] for j in range(6)) for i in range(64)] + [b"abbabaabba"]   # T = 9
        w0, w1, n_streams = 8, 4, 700
    else:
        keys = sorted({bytes(rng.choice(ab, size=int(rng.integers(3, 10)))) for _ in range(20)})
        w0, w1, n_streams = 7, 9, 800
    A = synth.build_automaton(keys)
    first = rng.choice(ab, size=(n_streams, w0))
    second = rng.choice(ab, size=(n_streams, w1))
    want = []
    if name == "seam":
        O = _oracle(keys)
        for s in range(n_streams):
            want += [(s, e - w0, k) for e, k in O.find_all(first[s].tobytes() + second[s].tobytes()) if e >= w0]
    else:
        for s in range(n_streams):
            it = A.iter_long(first[s].tobytes())
            list(it)
            it.set(second[s].tobytes())
            want += [(s, e - w0, k) for e, k in it]
    off = np.arange(n_streams + 1, dtype=np.int64) * w1
    return A, N.ALGO_LONG if name == "long_states" else N.ALGO_FILTER, first, (second.reshape(-1).copy(), off), want


FEED_KERNELS = ["seam", "long_states"]
KERNELS = ["pair", "pair_multi", "narrow", "wide", "dfa", "long"] + FEED_KERNELS
CAPS = ["0", "1", "31", "32", "33", "64", "65", "n-1", "n", "n+1"]
_cases = {}


def _cached(name, monkeypatch):
    if name not in _cases:
        _cases[name] = _feed_case(name) if name in FEED_KERNELS else _case(name, monkeypatch)
    return _cases[name]


def _write(kernel, A, algo, first, t, off, d_out, c, d_cnt, stream):
    """one scan (or, for a stream-batch site, a fresh batch's second feed) into d_out with capacity c"""
    import torch
    lib, tb = N.lib(), A._ensure_table(0)
    d_hay = torch.from_numpy(t).cuda()
    d_off = torch.from_numpy(off).cuda()
    if kernel not in FEED_KERNELS:
        N.check(lib.acb_scan_device(tb, d_hay.data_ptr(), t.size, d_off.data_ptr(), len(off) - 1, 0,
                                    d_out.data_ptr() if c else None, c, d_cnt.data_ptr(), stream.cuda_stream, algo))
        return
    ss = ctypes.c_void_p()
    N.check(lib.acb_streams_new(tb, len(first), int(kernel == "long_states"), ctypes.byref(ss)))
    try:
        found = ctypes.c_int64(0)
        N.check(lib.acb_streams_feed_host(ss, tb, N.ptr(first), first.size, None, len(first), first.shape[1], None,
                                          None, 1 << 16, ctypes.byref(found), algo, 1))
        N.check(lib.acb_streams_feed_device(ss, tb, d_hay.data_ptr(), t.size, d_off.data_ptr(), len(off) - 1, 0, None,
                                            d_out.data_ptr() if c else None, c, d_cnt.data_ptr(), stream.cuda_stream, algo))
        stream.synchronize()
    finally:
        lib.acb_streams_free(ss)


@pytest.mark.gpu
@pytest.mark.parametrize("cap", CAPS, ids=[f"cap{c}" for c in CAPS])
@pytest.mark.parametrize("kernel", KERNELS)
def test_scan_device_never_writes_past_cap(kernel, cap, monkeypatch):
    import torch
    A, algo, t, off, want = _cached(kernel, monkeypatch)
    first = None
    if kernel in FEED_KERNELS:
        first, (t, off) = t, off
    n = len(want)
    assert n > 200
    c = {"n-1": n - 1, "n": n, "n+1": n + 1}[cap] if cap.startswith("n") else int(cap)
    d_cnt = torch.zeros(1, dtype=torch.int64, device="cuda")
    d_out = torch.full((c + GUARD, 3), -1, dtype=torch.int32, device="cuda")
    stream = torch.cuda.current_stream()
    _write(kernel, A, algo, first, t, off, d_out, c, d_cnt, stream)
    stream.synchronize()
    out = d_out.cpu().numpy()
    assert (out[c:] == -1).all(), f"{int((out[c:] != -1).any(axis=1).sum())} guard rows written"
    assert int(d_cnt.item()) == n
    kept = _tuples(out[:min(c, n)])
    assert len(set(kept)) == len(kept)
    assert set(kept) <= set(want)
    if c >= n:
        assert sorted(kept) == sorted(want)


def _scan_host(A, algo, flat, off, cap, sort=1, room=None):
    """acb_scan_host into a caller buffer of cap + GUARD rows filled with -1: (rc, n_found, buffer)"""
    tb = A._ensure_table(0)
    out = np.full(((cap if room is None else room) + GUARD, 3), -1, dtype=np.int32)
    found = ctypes.c_int64(-1)
    rc = N.lib().acb_scan_host(tb, N.ptr(flat), flat.size, N.ptr(off), len(off) - 1, 0, N.ptr(out), cap,
                               ctypes.byref(found), algo, sort)
    return rc, found.value, out


def _check_host_bounds(A, algo, flat, off, want):
    n = len(want)
    rc, found, out = _scan_host(A, algo, flat, off, n - 1)
    assert rc == N.ACB_EOVERFLOW and found == n
    assert (out == -1).all()                                        # nothing is copied out on overflow
    rc, found, out = _scan_host(A, algo, flat, off, n)
    assert rc == N.ACB_OK and found == n
    assert _tuples(out[:n]) == want
    assert (out[n:] == -1).all()
    rc, found, out = _scan_host(A, algo, flat, off, n, sort=0, room=n + 5)
    assert rc == N.ACB_OK and sorted(_tuples(out[:n])) == sorted(want) and (out[n:] == -1).all()


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", ["pair", "narrow", "dfa", "long"])
def test_scan_host_overflow_is_exact_monolithic(kernel, monkeypatch):
    A, algo, t, off, want = _cached(kernel, monkeypatch)
    if kernel == "long":                                            # one haystack's records in increasing end_index
        want = sorted(want)
    _check_host_bounds(A, algo, t, off, want)


@pytest.mark.gpu
def test_scan_host_overflow_is_exact_pipelined():
    """64 MiB: the host scan runs as a pipeline over 32 MiB chunks, each sorted by itself"""
    rng = np.random.Generator(np.random.PCG64(4242))
    keys = synth.draw_keys(rng, synth.ALNUM, 600, 4, 16)
    A = synth.build_automaton(keys)
    flat, off = _big_batch(rng, keys, 64 * MiB + 77)
    want = _tuples(_oracle(keys).scan_batch_bytes(flat, off))
    assert len(want) > 8192
    lib = N.lib()
    A._ensure_table(0)
    before = lib.acb_launch_count()
    rc, found, _ = _scan_host(A, N.ALGO_FILTER, flat, off, len(want))
    assert rc == N.ACB_OK and lib.acb_launch_count() - before >= 4         # 3 chunks: a scan and a sort each
    _check_host_bounds(A, N.ALGO_FILTER, flat, off, want)
    fresh = synth.build_automaton(keys)                                     # 4096 records: the first attempt overflows
    m = fresh.find_all_batch((flat, off))
    assert fresh._match_cap > 4096
    assert triples(m) == want


# ------------------------------------------------------------------ the record sort, called directly
SORT_N_HAY = [2, 1 << 16, (1 << 16) + 1, (1 << 31) - 1]
SORT_LETTERS = [1, (1 << 20) - 1, 1 << 20, (1 << 31) - 1]
SORT_LEN = [1, 3, 4, 7, 8]                      # bits_for: 1, 2, 3, 3, 4; with 31 + 31 bits, 3 is 64 bits and 4 is 65


def _sort_automaton(max_len):
    """keys of every length 1..max_len, two of each: equal sort keys with different key ids (stability)"""
    A = ac.flavour("bytes").Automaton(ac.STORE_INTS)
    for ln in range(1, max_len + 1):
        A.add_word(b"a" * ln, 2 * ln - 2)
        A.add_word(b"b" * ln, 2 * ln - 1)
    A.make_automaton()
    return A


def _synthetic_records(rng, n, n_hay, max_letters, n_keys):
    rec = np.empty((n, 3), dtype=np.int32)
    rec[:, 0] = rng.integers(0, n_hay, size=n)
    rec[:, 1] = rng.integers(0, max_letters, size=n)
    rec[:, 2] = rng.integers(0, n_keys, size=n)
    rec[:5, 0] = n_hay - 1                                          # the top of every field
    rec[5:10, 1] = max_letters - 1
    rec[10:400, :2] = rec[400:790, :2]                              # ties in (hay, end): the length decides, then the input order
    if n_hay > 2:
        rec[790:800, 0] = 1 << (bits_for(n_hay - 1) - 1)           # the highest bit of hay_id
    return rec


_sort_tables = {}


@pytest.mark.gpu
@pytest.mark.parametrize("max_len", SORT_LEN)
@pytest.mark.parametrize("max_letters", SORT_LETTERS)
@pytest.mark.parametrize("n_hay", SORT_N_HAY)
def test_sort_matches_device_at_field_boundaries(n_hay, max_letters, max_len):
    import torch
    if max_len not in _sort_tables:
        _sort_tables[max_len] = _sort_automaton(max_len)
    A = _sort_tables[max_len]
    tb = A._ensure_table(0)
    kl = np.asarray(A.flat()["key_len"], dtype=np.int64)
    assert kl.max() == max_len
    rng = np.random.Generator(np.random.PCG64(n_hay * 31 + max_letters * 7 + max_len))
    rec = _synthetic_records(rng, 3000, n_hay, max_letters, len(kl))
    d = torch.from_numpy(rec).cuda()
    stream = torch.cuda.current_stream()
    rc = N.lib().acb_sort_matches_device(tb, d.data_ptr(), len(rec), n_hay, max_letters, stream.cuda_stream)
    stream.synchronize()
    got = d.cpu().numpy()
    if sort_bits(n_hay, max_letters, max_len) > 64:
        assert rc == N.ACB_ERANGE and np.array_equal(got, rec)
        return
    assert rc == N.ACB_OK
    want = rec[np.lexsort((-kl[rec[:, 2]], rec[:, 1], rec[:, 0]))]   # lexsort is stable, as the radix sort is
    assert np.array_equal(got, want)


def test_sort_boundary_cases_are_on_both_sides_of_64_bits():
    """the grid above has a sort key of exactly 64 bits (top hay_id bit in use) and one of 65"""
    assert sort_bits((1 << 31) - 1, (1 << 31) - 1, 3) == 64
    assert sort_bits((1 << 31) - 1, (1 << 31) - 1, 4) == 65
    assert sort_bits((1 << 16) + 1, 1 << 20, 8) == 17 + 21 + 4


@pytest.mark.gpu
def test_sort_matches_device_zero_and_one_record():
    import torch
    A = _sort_automaton(3)
    tb = A._ensure_table(0)
    stream = torch.cuda.current_stream()
    one = torch.tensor([[5, 6, 1]], dtype=torch.int32, device="cuda")
    assert N.lib().acb_sort_matches_device(tb, None, 0, 10, 10, stream.cuda_stream) == N.ACB_OK
    assert N.lib().acb_sort_matches_device(tb, one.data_ptr(), 1, 10, 10, stream.cuda_stream) == N.ACB_OK
    stream.synchronize()
    assert one.cpu().tolist() == [[5, 6, 1]]


@pytest.mark.gpu
def test_sort_matches_device_on_two_streams():
    """two sorts of different record sets for one table, issued on two CUDA streams with no host wait between them: the
    second waits for the first before it reuses the table's sort scratch.  Without that wait the second would overwrite
    keys the first may still be reading; whether the first is still running then is up to the device, so the test can
    pass without the wait too."""
    import torch
    A = _sort_automaton(4)
    tb = A._ensure_table(0)
    kl = np.asarray(A.flat()["key_len"], dtype=np.int64)
    n_hay, max_letters = 1 << 16, (1 << 20) - 1
    rng = np.random.Generator(np.random.PCG64(5))
    recs = [_synthetic_records(rng, n, n_hay, max_letters, len(kl)) for n in (400_000, 300_000)]
    ds = [torch.from_numpy(r).cuda() for r in recs]
    torch.cuda.synchronize()
    for d, s in zip(ds, (torch.cuda.Stream(), torch.cuda.Stream())):
        N.check(N.lib().acb_sort_matches_device(tb, d.data_ptr(), len(d), n_hay, max_letters, s.cuda_stream))
    torch.cuda.synchronize()
    for d, r in zip(ds, recs):
        assert np.array_equal(d.cpu().numpy(), r[np.lexsort((-kl[r[:, 2]], r[:, 1], r[:, 0]))])


# ------------------------------------------------------------------ the record sort through its callers
def _one_long_key_batch(long_letters, rng):
    """about 128 MiB in 65 536 haystacks; keys: one of `long_letters` letters (it never matches) and short keys that
    end together (the order inside one end index is longest first)"""
    short = [b"wxyz", b"xyz", b"yz", b"zz", b"qwxy"]
    long_key = bytes(rng.choice(np.frombuffer(b"abcd", dtype=np.uint8), size=long_letters))
    keys = short + [long_key]
    n = 128 * MiB
    flat = rng.choice(np.frombuffer(b"efghijklmnop", dtype=np.uint8), size=n)
    for i, b in enumerate(range(50, n - 8, 2039)):
        k = short[i % 4] if i % 3 else b"qwxyz"
        flat[b:b + len(k)] = np.frombuffer(k, dtype=np.uint8)
    off = np.concatenate([[0], np.sort(rng.integers(0, n, size=65535)), [n]]).astype(np.int64)
    return keys, flat, off


@pytest.mark.gpu
@pytest.mark.parametrize("log_len", [19, 20])
def test_sort_key_width_selects_the_host_route(log_len):
    """2^19 letters: the sort key is exactly 64 bits, the batch goes through the pipelined route with a device sort per
    chunk; 2^20: 65 bits, the monolithic route with its std::sort fallback.  Both must equal the oracle."""
    rng = np.random.Generator(np.random.PCG64(log_len))
    keys, flat, off = _one_long_key_batch(1 << log_len, rng)
    bits = sort_bits(len(off) - 1, flat.size, 1 << log_len)
    assert bits == (64 if log_len == 19 else 65)
    A = synth.build_automaton(keys)
    want = _tuples(_oracle(keys).scan_batch_bytes(flat, off))
    assert len(want) > 100_000
    lib = N.lib()
    A._ensure_table(0)
    A._match_cap = len(want)
    before = lib.acb_launch_count()
    m = A.find_all_batch((flat, off), algo="filter")
    launches = lib.acb_launch_count() - before
    assert launches == (8 if log_len == 19 else 1)          # 4 chunks: scan + sort each / one scan, sorted on the host
    got = triples(m)
    assert got == want


@pytest.mark.gpu
def test_device_tensor_entry_sorts_on_the_host_when_the_device_sort_refuses(monkeypatch):
    """_scan_device_tensor falls back to np.lexsort on ACB_ERANGE (a fixed-stride batch that needs it cannot be
    allocated, so the library call is wrapped)"""
    import torch
    keys = [b"abcd", b"bcd", b"cd", b"d", b"ab", b"xab"]
    A = synth.build_automaton(keys)
    rng = np.random.Generator(np.random.PCG64(77))
    rows = rng.choice(np.frombuffer(b"abcdx", dtype=np.uint8), size=(300, 64))
    want = _tuples(_oracle(keys).scan_batch_bytes(rows.reshape(-1), np.arange(301, dtype=np.int64) * 64))
    calls = []

    def refuse(*a):
        calls.append(a[2])
        return N.ACB_ERANGE
    monkeypatch.setattr(N.lib(), "acb_sort_matches_device", refuse)
    m = A.find_all_batch(torch.from_numpy(rows).cuda())
    assert calls == [len(want)]
    assert triples(m) == want
