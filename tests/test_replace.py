"""Replacer.replace_batch / acb_replace_device / acb_replace_host: every leftmost-longest match replaced, on the GPU.

The answer is always emul_replace.definition over the matches the definition of the selection (emul_leftmost.greedy)
takes from the C oracle's full list, or, at scale, a numpy build from find_leftmost_longest_batch's records.  The CPU
tests run the numpy restatement of both passes (tests/emul_replace.py) at tiny tile sizes; the gpu-marked tests run the
real kernels."""
import ctypes

import numpy as np
import pytest

import emul_leftmost
import emul_replace
import pyahocorasick_b200 as pkg
from batch_cases import (CASES, DT, NESTED, automaton, fake_table, forms, layout, leftmost_random_case,
                         leftmost_structured_cases, obj, oracle_full, replace_reps, rows, skip_if_device, split,
                         table_and_batch)
from pyahocorasick_b200 import _native as N

TILES = [1, 3, 16, 64]
WIDTH = {"bytes": 1, "latin1": 1, "wide": 4, "mixed": 4, "seq2": 2, "seq4": 4}


def _want(O, keys, hays, reps, case="bytes"):
    """per haystack, the definition over the selection's definition over the oracle's full list"""
    chosen = [[] for _ in hays]
    for h, e, k in emul_leftmost.greedy(oracle_full(O, hays, case), [len(k) for k in keys]):
        chosen[h].append((e, k))
    return [emul_replace.definition(h, c, [len(k) for k in keys], reps) for h, c in zip(hays, chosen)]


def _restated(O, keys, hays, reps, case, tile):
    w = WIDTH[case]
    flat, offs = layout(hays, w)
    kl = np.array([len(k) for k in keys])
    chosen = np.array(emul_leftmost.greedy(oracle_full(O, hays, case), kl), dtype=np.int64).reshape(-1, 3)
    rep, rep_off = layout(reps, w)
    out, out_off = emul_replace.replace(flat, offs, chosen, kl, rep, rep_off, w, tile)
    return split(out, out_off, w)


# ------------------------------------------------------------------ the restatement against the definition (CPU)
def _structured_reps(keys):
    """empty, shorter, equal and longer replacements, and one that holds keys"""
    return [[], list(keys[0]) * 3, list(keys[-1][:1]), list(keys[0]) + [0x7A]] * (len(keys) // 4 + 1)


@pytest.mark.parametrize("tile", TILES)
def test_restatement_equals_the_definition_on_the_oracle(tile):
    rng = np.random.default_rng(tile)
    for case, (fl, seq, _) in CASES.items():
        for _ in range(10):
            keys, hays = leftmost_random_case(case, rng)
            _, O = automaton(fl, seq, keys)
            reps = replace_reps(case, keys, rng)
            assert _restated(O, keys, hays, reps, case, tile) == _want(O, keys, hays, reps, case), (case, keys, hays, reps)
    for keys, hays in list(leftmost_structured_cases()) + [(NESTED, [[0x61] * 100, [], [], [0x62] * 40, [0x61, 0x62] * 30])]:
        _, O = automaton("bytes", False, keys)
        reps = _structured_reps(keys)[:len(keys)]
        assert _restated(O, keys, hays, reps, "bytes", tile) == _want(O, keys, hays, reps)


@pytest.mark.parametrize("tile", [1, 16])
def test_python_layer_on_the_restatement(monkeypatch, tile):
    """every input form, the mapping mode on STORE_INTS, the values mode on STORE_ANY"""
    emul_replace.install(monkeypatch, tile)
    rng = np.random.default_rng(30 + tile)
    for case, (fl, seq, _) in CASES.items():
        for _ in range(4):
            keys, hays = leftmost_random_case(case, rng)
            A, O = automaton(fl, seq, keys)
            reps = replace_reps(case, keys, rng)
            want = _want(O, keys, hays, reps, case)
            R = A.replacer({obj(fl, seq, k): obj(fl, seq, r) for k, r in zip(keys, reps)})
            for form, batch in forms([obj(fl, seq, h) for h in hays], hays, A._L, case in ("latin1", "mixed")):
                got = R.replace_batch(batch)
                if form == "list":
                    assert got == [obj(fl, seq, h) for h in want], (case, form)
                else:
                    out, offs = got
                    assert offs.dtype == np.int64 and split(out, offs, A._L) == want, (case, form)
            mod = pkg.flavour(fl)
            B = mod.Automaton(mod.STORE_ANY, mod.KEY_SEQUENCE) if seq else mod.Automaton(mod.STORE_ANY)
            for k, r in zip(keys, reps):
                B.add_word(obj(fl, seq, k), obj(fl, seq, r))
            B.make_automaton()
            assert B.replacer().replace_batch([obj(fl, seq, h) for h in hays]) == [obj(fl, seq, h) for h in want], case


def test_latin1_table_only_when_every_replacement_is_latin1(monkeypatch):
    emul_replace.install(monkeypatch)
    seen = []
    run = pkg.automaton.Replacer._run_host

    def spy(self, flat, offs, n, narrow, algo):
        seen.append(narrow)
        return run(self, flat, offs, n, narrow, algo)

    monkeypatch.setattr(pkg.automaton.Replacer, "_run_host", spy)
    A = pkg.flavour("unicode").Automaton()
    for k in ("ab", "é", "bł"):
        A.add_word(k, k)
    A.make_automaton()
    hays = ["xabéy", "", "ébab"]
    R = A.replacer({"ab": "AB", "é": "", "bł": "Z"})
    assert R.replace_batch(hays) == ["xABy", "", "bAB"] and seen == [True]
    R = A.replacer({"ab": "\U0001F600", "é": "", "bł": "Z"})
    assert R.replace_batch(hays) == ["x\U0001F600y", "", "b\U0001F600"] and seen == [True, False]
    assert R.replace_batch(["abł", "\ud800ab"]) == ["\U0001F600ł", "\ud800\U0001F600"] and seen[-1] is False


def test_errors_stale_and_snapshot(monkeypatch):
    emul_replace.install(monkeypatch)
    mod = pkg.flavour("bytes")
    A = mod.Automaton()
    A.add_word(b"ab", b"X")
    with pytest.raises(AttributeError):
        A.replacer()                                           # not built: what find_all_batch raises
    A.add_word(b"cd", b"Y")
    A.make_automaton()
    with pytest.raises(KeyError) as e:
        A.replacer({b"cd": b""})
    assert e.value.args == (b"ab",)                            # the first missing key in insertion order
    with pytest.raises(TypeError):
        A.replacer({b"ab": "str", b"cd": b""})
    R = A.replacer({b"ab": b"1", b"cd": b"2", b"zz": 5})        # entries for keys that are not live are ignored
    with pytest.raises(ValueError):
        R.replace_batch([b"ab"], algo="long")
    assert R.replace_batch([b"xabcd"]) == [b"x12"]
    V = A.replacer()
    A.add_word(b"ab", b"new value")                            # same key: the version does not move ...
    assert V._tables[False][0].tobytes() == b"XY"              # ... and the replacer keeps its snapshot
    with pytest.raises(AttributeError):
        V.replace_batch([b"ab"])                               # not built again: what find_all_batch raises
    A.make_automaton()
    assert A.replacer().replace_batch([b"ab"]) == [b"new value"]
    for r in (R, V):
        with pytest.raises(ValueError):
            r.replace_batch([b"ab"])                           # stale
    W = A.replacer()
    A.add_word(b"ef", b"Z")
    with pytest.raises(ValueError):
        W.replace_batch([b"ab"])                               # a new key: stale
    I = mod.Automaton(mod.STORE_INTS)
    I.add_word(b"ab", 1)
    I.make_automaton()
    with pytest.raises(ValueError):
        I.replacer()                                           # values are ints: a mapping is needed
    assert I.replacer({b"ab": b""}).replace_batch([b"aabb"]) == [b"ab"]
    S = mod.Automaton(mod.STORE_INTS, mod.KEY_SEQUENCE)
    S.add_word((1, 2), 0)
    S.make_automaton()
    with pytest.raises(ValueError):
        S.replacer({(1, 2): (70000,)})                         # a 2-byte letter out of range
    with pytest.raises(TypeError):
        S.replacer({(1, 2): b"x"})
    assert S.replacer({(1, 2): (9, 9, 9)}).replace_batch([(0, 1, 2, 3)]) == [(0, 9, 9, 9, 3)]


def test_every_key_removed_gives_the_input(monkeypatch):
    emul_replace.install(monkeypatch)
    A = pkg.flavour("bytes").Automaton()
    A.add_word(b"ab", b"")
    A.remove_word(b"ab")
    A.add_word(b"q", b"")
    A.remove_word(b"q")
    A.make_automaton()
    if A.kind != pkg.AHOCORASICK:
        pytest.skip("an empty key set does not build")
    hays = [b"abq", b"", b"ab"]
    assert A.replacer().replace_batch(hays) == hays


def test_c_entries_check_arguments_first():
    L = N.lib()
    tb = fake_table(1)
    rep = np.frombuffer(b"xyz", dtype=np.uint8)
    r = ctypes.c_void_p()
    bad_offsets = ([1, 3], [0, 2], [0, 4], [0, 2, 1, 3])
    assert L.acb_replacer_new(None, N.ptr(rep), 3, N.ptr(np.array([0, 3], np.int64)), 1, ctypes.byref(r)) == N.ACB_EINVAL
    assert L.acb_replacer_new(ctypes.addressof(fake_table(0)), N.ptr(rep), 3, N.ptr(np.array([0, 3], np.int64)), 1,
                              ctypes.byref(r)) == N.ACB_EINVAL
    for offs in bad_offsets:
        o = np.array(offs, dtype=np.int64)
        assert L.acb_replacer_new(ctypes.addressof(tb), N.ptr(rep), 3, N.ptr(o), len(o) - 1, ctypes.byref(r)) == N.ACB_EINVAL, offs
    o = np.array([0, 2, 4], np.int64)
    assert L.acb_replacer_new(ctypes.addressof(fake_table(2)), N.ptr(rep), 3, N.ptr(o), 2, ctypes.byref(r)) == N.ACB_EINVAL
    fake_r = fake_table(0)                                     # a zeroed replacer: letter width 0 does not fit the table
    hay = np.zeros(32, dtype=np.uint8)
    offs = np.array([0, 16, 32], np.int64)
    out_offs = np.zeros(3, np.int64)
    total = ctypes.c_int64(0)
    args = (N.ptr(hay), 32, N.ptr(offs), 2, 0, N.ALGO_AUTO, N.ptr(out_offs), N.ptr(hay), 32, ctypes.byref(total))
    assert L.acb_replace_host(ctypes.addressof(fake_r), ctypes.addressof(tb), *args) == N.ACB_EINVAL
    assert L.acb_replace_host(None, ctypes.addressof(tb), *args) == N.ACB_EINVAL
    cnt = np.zeros(1, np.int64)
    assert L.acb_replace_device(None, ctypes.addressof(tb), N.ptr(hay), 32, None, 2, 16, None, 0, N.ptr(cnt), N.ptr(out_offs),
                                None, 0, N.ptr(cnt), None) == N.ACB_EINVAL
    ms = (ctypes.c_float * 2)()
    assert L.acb_last_replace_ms(ms, 3) == N.ACB_EINVAL and L.acb_last_replace_ms(ms, 2) == N.ACB_OK


def test_c_entries_fail_loudly_without_a_device():
    skip_if_device()
    tb = fake_table(1)
    rep = np.frombuffer(b"xyz", dtype=np.uint8)
    r = ctypes.c_void_p()
    assert N.lib().acb_replacer_new(ctypes.addressof(tb), N.ptr(rep), 3, N.ptr(np.array([0, 3], np.int64)), 1,
                                    ctypes.byref(r)) == N.ACB_ECUDA
    assert N.last_error()


# ------------------------------------------------------------------ the real kernels
@pytest.mark.gpu
@pytest.mark.parametrize("algo", ["filter", "dfa"])
def test_gpu_fuzz_against_the_definition(algo):
    rng = np.random.default_rng(41)
    for case, (fl, seq, _) in CASES.items():
        for _ in range(6):
            keys, hays = leftmost_random_case(case, rng)
            A, O = automaton(fl, seq, keys)
            reps = replace_reps(case, keys, rng)
            want = _want(O, keys, hays, reps, case)
            R = A.replacer({obj(fl, seq, k): obj(fl, seq, r) for k, r in zip(keys, reps)})
            for form, batch in forms([obj(fl, seq, h) for h in hays], hays, A._L, case in ("latin1", "mixed")):
                got = R.replace_batch(batch, algo=algo)
                if form == "list":
                    assert got == [obj(fl, seq, h) for h in want], (case, form, keys, hays)
                else:
                    assert split(*got, A._L) == want, (case, form)
    for keys, hays in leftmost_structured_cases():
        A, O = automaton("bytes", False, keys)
        reps = _structured_reps(keys)[:len(keys)]
        R = A.replacer({bytes(k): bytes(r) for k, r in zip(keys, reps)})
        assert R.replace_batch([bytes(h) for h in hays], algo=algo) == [bytes(h) for h in _want(O, keys, hays, reps)]


def _np_replace(flat, in_off, chosen, key_len, rep, rep_off):
    """the whole output of a bytes batch from its chosen records (hay, end, key), vectorised -> (bytes, offsets)"""
    chosen = np.asarray(chosen, dtype=np.int64).reshape(-1, 3)
    hay, end, key = chosen[:, 0], chosen[:, 1], chosen[:, 2]
    ln, rl = key_len[key], rep_off[key + 1] - rep_off[key]
    s = in_off[hay] + end - ln + 1
    cov = np.zeros(flat.size + 1, dtype=np.int64)
    np.add.at(cov, s, 1)
    np.add.at(cov, s + ln, -1)
    keep = np.cumsum(cov[:-1]) == 0                            # input bytes that are copied
    units = keep.astype(np.int64)                              # output bytes per input byte
    units[s] += rl                                             # a match's first byte carries its replacement
    pos = np.zeros(flat.size + 1, dtype=np.int64)
    np.cumsum(units, out=pos[1:])
    out = np.empty(int(pos[-1]), dtype=np.uint8)
    out[pos[:-1][keep]] = flat[keep]
    j = np.arange(int(rl.sum())) - np.repeat(np.cumsum(rl) - rl, rl)
    out[np.repeat(pos[s], rl) + j] = rep[np.repeat(rep_off[key], rl) + j]
    return out, pos[in_off]


def _check_batch(A, table, flat, offs, tensor=None):
    """replace_batch from the host pair (and from a CUDA tensor) against _np_replace over the selection's records"""
    import torch
    kl = np.asarray(A.flat()["key_len"], dtype=np.int64)
    rep, rep_off = emul_replace_layout(A, table)
    chosen = rows(A.find_leftmost_longest_batch((flat, offs)))
    want, want_off = _np_replace(flat, offs, chosen, kl, rep, rep_off)
    R = A.replacer(table)
    out, out_off = R.replace_batch((flat, offs))
    assert np.array_equal(out_off, want_off) and np.array_equal(out, want)
    if tensor is not None:
        o, oo = R.replace_batch(tensor)
        assert oo.is_cuda and o.is_cuda
        assert np.array_equal(oo.cpu().numpy(), want_off) and torch.equal(o.cpu(), torch.from_numpy(want))
    return want, want_off


def emul_replace_layout(A, table):
    reps = [b""] * len(A._key_objs)
    for kid, k in enumerate(A._key_objs):
        if k is not None:
            reps[kid] = table[k]
    offs = np.zeros(len(reps) + 1, dtype=np.int64)
    np.cumsum([len(r) for r in reps], out=offs[1:])
    return np.frombuffer(b"".join(reps) or b"\0", dtype=np.uint8), offs


@pytest.mark.gpu
def test_gpu_c2_planted_whole_output():
    """C2 (1 M x 256 B, one planted key each): random replacement lengths 0..24, the identity, and delete-everything"""
    import torch
    from pyahocorasick_b200 import synth
    w = synth.make("C2")
    A = synth.build_automaton(w.keys)
    rng = np.random.default_rng(8)
    d = torch.from_numpy(w.haystacks).cuda()
    flat = w.haystacks.reshape(-1)
    offs = np.arange(w.n_hay + 1, dtype=np.int64) * w.haystacks.shape[1]
    keys = [k for k in A._key_objs if k is not None]
    lens = rng.integers(0, 25, size=len(keys))
    table = {k: bytes(rng.integers(0, 256, size=int(n), dtype=np.uint8)) for k, n in zip(keys, lens)}
    want, _ = _check_batch(A, table, flat, offs, d)
    assert want.size != flat.size
    ident, ident_off = _check_batch(A, {k: k for k in keys}, flat, offs, d)
    assert np.array_equal(ident, flat) and np.array_equal(ident_off, offs)
    gone, _ = _check_batch(A, {k: b"" for k in keys}, flat, offs)
    assert gone.size < flat.size


@pytest.mark.gpu
def test_gpu_tile_and_segment_boundaries():
    """one 64 MiB haystack of abutting matches of lengths 1..33 with replacements of 0..33 bytes, so that segment ends
    fall at every residue around every tile and 16-byte boundary; a 1 MiB gap, a 200 KiB replacement, runs of empty
    haystacks across a tile"""
    rng = np.random.default_rng(12)
    keys = [bytes([0x41 + i]) * (i + 1) for i in range(33)] + [b"#big#"]
    A, _ = automaton("bytes", False, keys)
    table = {k: bytes(rng.integers(0x61, 0x7B, size=int(rng.integers(0, 34)), dtype=np.uint8)) for k in keys[:33]}
    table[keys[0]] = b""
    table[b"#big#"] = bytes(rng.integers(0, 256, size=200 << 10, dtype=np.uint8))
    pick = rng.integers(0, 33, size=(64 << 20) // 17)
    body = b"".join(keys[i] for i in pick.tolist())
    text = body[: 32 << 20] + b"." * (1 << 20) + b"#big#" + body[32 << 20:]
    flat = np.frombuffer(text, dtype=np.uint8)
    cuts = [0] + [len(text) // 2 + 7] * 3000 + [len(text) // 2 + 9] * 5 + [len(text)]
    offs = np.array(cuts, dtype=np.int64)
    _check_batch(A, table, flat, offs)


@pytest.mark.gpu
def test_gpu_output_past_2_gib():
    """a CUDA batch whose output passes 2^31 bytes (32 x 4 MiB of 'ab' -> 40 bytes each), and one haystack whose own
    output does (64 MiB of 'ab' -> 72 bytes each); checked on the device"""
    import torch
    A, _ = automaton("bytes", False, [list(b"ab"), list(b"zz")])
    for rows, stride, rl in ((32, 4 << 20, 40), (1, 64 << 20, 72)):
        rep = bytes(range(1, rl + 1))
        d = torch.tensor(list(b"ab"), dtype=torch.uint8, device="cuda").repeat(rows * stride // 2).view(rows, stride)
        out, offs = A.replacer({b"ab": rep, b"zz": b""}).replace_batch(d)
        per = stride // 2 * rl
        assert out.numel() == rows * per and out.numel() > (1 << 31)
        assert torch.equal(offs.cpu(), torch.arange(rows + 1, dtype=torch.int64) * per)
        assert bool((out.view(-1, rl) == torch.tensor(list(rep), dtype=torch.uint8, device="cuda")).all())
        del out, d
        torch.cuda.empty_cache()


@pytest.mark.gpu
def test_gpu_capacity_contract():
    import torch
    keys = [b"ab", b"b", b"abc"]
    A, _ = automaton("bytes", False, keys)
    table = {b"ab": b"XYZW", b"b": b"", b"abc": b"q"}
    hays = [b"abcabxbab" * 20, b"", b"bbbb", b"zzz"]
    tb, flat, offs = table_and_batch(A, hays)
    want, want_off = _check_batch(A, table, flat, offs)
    total = int(want_off[-1])
    L = N.lib()
    R = A.replacer(table)
    r = R._replacer(tb, False, 0)
    got_off = np.zeros(len(hays) + 1, dtype=np.int64)
    t = ctypes.c_int64(0)
    for cap in (0, total - 1, total):
        buf = np.full(cap + 64, 0xEE, dtype=np.uint8)
        rc = L.acb_replace_host(r, tb, N.ptr(flat), flat.size, N.ptr(offs), len(hays), 0, N.ALGO_AUTO, N.ptr(got_off),
                                N.ptr(buf), cap, ctypes.byref(t))
        assert rc == (N.ACB_OK if cap >= total else N.ACB_EOVERFLOW) and t.value == total
        assert np.array_equal(got_off, want_off)
        if cap >= total:
            assert np.array_equal(buf[:total], want)
        assert (buf[min(cap, total) if cap >= total else 0:] == 0xEE).all()
    # the device entry, on records the selection left on the device
    d = torch.from_numpy(flat.copy()).cuda()
    d_off = torch.from_numpy(offs).cuda()
    chosen = torch.from_numpy(rows(A.find_leftmost_longest_batch((flat, offs))).astype(np.int32)).cuda()
    n = torch.tensor([chosen.shape[0]], dtype=torch.int64, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    for cap in (0, total - 1, total):
        out = torch.full((total + 64,), 0xEE, dtype=torch.uint8, device="cuda")
        oo = torch.full((len(hays) + 1,), -1, dtype=torch.int64, device="cuda")
        tt = torch.full((1,), -1, dtype=torch.int64, device="cuda")
        assert L.acb_replace_device(r, tb, d.data_ptr(), flat.size, d_off.data_ptr(), len(hays), 0, chosen.data_ptr(),
                                    chosen.shape[0], n.data_ptr(), oo.data_ptr(), out.data_ptr(), cap, tt.data_ptr(), s) == N.ACB_OK
        assert int(tt.item()) == total and np.array_equal(oo.cpu().numpy(), want_off)
        o = out.cpu().numpy()
        if cap >= total:
            assert np.array_equal(o[:total], want) and (o[total:] == 0xEE).all()
        else:
            assert (o == 0xEE).all()                           # nothing written when the output does not fit
    assert L.acb_replace_device(r, tb, d.data_ptr() + 1, flat.size - 1, None, 1, flat.size - 1, chosen.data_ptr(), 0, n.data_ptr(),
                                oo.data_ptr(), out.data_ptr(), 0, tt.data_ptr(), s) == N.ACB_EINVAL


@pytest.mark.gpu
@pytest.mark.parametrize("fl", ["bytes", "unicode"])
def test_gpu_cuda_tensors_on_a_side_stream(fl):
    import torch
    rng = np.random.default_rng(15)
    case = "bytes" if fl == "bytes" else "wide"
    al = CASES[case][2]
    keys = sorted({tuple(int(x) for x in rng.choice(al[:2], size=int(rng.integers(1, 5)))) for _ in range(10)})
    A, O = automaton(*CASES[case][:2], keys)
    reps = replace_reps(case, keys, rng)
    R = A.replacer({obj(*CASES[case][:2], k): obj(*CASES[case][:2], r) for k, r in zip(keys, reps)})
    hays = [[int(x) for x in rng.choice(al, size=7)] for _ in range(300)]
    host = np.stack([np.asarray(h, dtype=DT[A._L]).view(np.uint8) for h in hays])
    d = torch.from_numpy(host).cuda()
    views = {"whole": (d, hays)}
    if A._L == 1:
        views["misaligned"] = (d[1:], hays[1:])
        assert d[1:].data_ptr() % 16 != 0
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    for name, (t, hs) in views.items():
        with torch.cuda.stream(side):
            out, offs = R.replace_batch(t)
        side.synchronize()
        assert split(out.cpu().numpy(), offs.cpu().numpy(), A._L) == _want(O, keys, hs, reps, case), name
