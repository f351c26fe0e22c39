"""encoding="utf-8" of find_all_batch, find_long_batch, find_leftmost_longest_batch, find_leftmost_first_batch and
Replacer.replace_batch: UTF-8 haystacks decoded to letters on the GPU, replacement output encoded back to UTF-8 there.

The CPU half checks the restatement of the per-byte rule (tests/emul_utf8.py) against CPython's decoder and the
refusals.  The gpu-marked half runs the C entries at both letter widths against the restatement, and every route,
input form and option against the same call on the decoded list of str."""
import ctypes
import itertools
import random

import numpy as np
import pytest

import emul_utf8 as eu
import pyahocorasick_b200 as pkg
from batch_cases import automaton, oracle_full, triples
from pyahocorasick_b200 import _native as N

TRAPS = [0x00, 0x41, 0x7F, 0x80, 0x8F, 0x90, 0x9F, 0xA0, 0xBF, 0xC0, 0xC1, 0xC2, 0xDF, 0xE0, 0xE1, 0xEC, 0xED, 0xEE,
         0xEF, 0xF0, 0xF1, 0xF3, 0xF4, 0xF5, 0xFF]
EDGES = [0x7F, 0x80, 0x8F, 0x90, 0x9F, 0xA0, 0xBF, 0xC0]
# the launches a UTF-8 batch adds to the decoded-str device route: decode pass 1 and its offsets, pass 2
DECODE_LAUNCHES = 3


def cpython(h: bytes):
    """("replace" text, strict (start, end) or None) from CPython"""
    try:
        h.decode("utf-8")
        err = None
    except UnicodeDecodeError as e:
        err = (e.start, e.end)
    return h.decode("utf-8", "replace"), err


def check_rule(h: bytes):
    text, err = cpython(h)
    assert eu.decode(h) == text, h
    assert eu.first_error(h) == err, h


def test_rule_two_bytes():
    for a in range(256):
        for b in range(256):
            check_rule(bytes([a, b]))


def test_rule_leads_and_boundary_continuations():
    for lead in range(256):
        for k in range(4):
            for tail in itertools.product(EDGES, repeat=k):
                check_rule(bytes([lead, *tail]))


def test_rule_fuzz():
    rng = random.Random(20)
    for _ in range(40000):
        check_rule(bytes(rng.choice(TRAPS) for _ in range(rng.randint(0, 12))))


def unicode_automaton(keys=("ab", "é", "€")):
    mod = pkg.flavour("unicode")
    A = mod.Automaton(mod.STORE_INTS)
    for i, k in enumerate(keys):
        A.add_word(k, i)
    A.make_automaton()
    return A


def test_refusals():
    A = unicode_automaton()
    hays = [b"ab", "é".encode()]
    for enc in ("latin-1", "utf-16", "utf-8-sig", "no-such-codec"):
        with pytest.raises(ValueError):
            A.find_all_batch(hays, encoding=enc)
    for errors in ("ignore", "surrogatepass", "backslashreplace"):
        with pytest.raises(ValueError):
            A.find_all_batch(hays, encoding="utf-8", errors=errors)
    with pytest.raises(ValueError):
        A.find_all_batch(hays, errors="replace")                      # errors without an encoding
    with pytest.raises(TypeError):
        A.find_all_batch([b"ab", "ab"], encoding="utf-8")
    with pytest.raises(TypeError):
        A.find_leftmost_longest_batch(["ab"], encoding="UTF8")
    with pytest.raises(TypeError):
        unicode_store_any(["ab"]).replacer({"ab": "x"}).replace_batch([b"x", 3], encoding="utf_8")
    B = pkg.flavour("bytes").Automaton(pkg.STORE_INTS)
    B.add_word(b"ab", 0)
    B.make_automaton()
    with pytest.raises(ValueError):
        B.find_all_batch([b"ab"], encoding="utf-8")
    mod = pkg.flavour("unicode")
    S = mod.Automaton(mod.STORE_INTS, mod.KEY_SEQUENCE)
    S.add_word((1, 2), 0)
    S.make_automaton()
    with pytest.raises(ValueError):
        S.find_long_batch([b"ab"], encoding="utf-8")


def test_no_encoding_keeps_letter_arrays():
    """a uint8 array without encoding is still 4-byte letters: rows must hold whole letters"""
    A = unicode_automaton()
    b = A._batch_input(np.zeros((2, 8), dtype=np.uint8))
    assert (b.kind, b.n, b.stride, b.narrow) == ("host", 2, 8, False)
    with pytest.raises(ValueError):
        A._batch_input(np.zeros((2, 6), dtype=np.uint8))


# ------------------------------------------------------------------------------------------------ GPU: the C entries
def _torch():
    import torch
    return torch


def c_decode(hays=None, rows=None, errors=N.UTF8_REPLACE, width=4):
    """the C entries on cuda:0: (letters per haystack at `width`, info block)"""
    torch = _torch()
    lib = N.lib()
    if rows is not None:
        flat, offs, n, stride = rows.reshape(-1), None, rows.shape[0], rows.shape[1]
    else:
        flat = np.frombuffer(b"".join(hays), dtype=np.uint8)
        offs = np.zeros(len(hays) + 1, dtype=np.int64)
        np.cumsum([len(h) for h in hays], out=offs[1:])
        n, stride = len(hays), 0
    t = torch.tensor(flat.copy(), device="cuda:0")
    d_off = None if offs is None else torch.from_numpy(offs).cuda()
    need = ctypes.c_int64(0)
    N.check(lib.acb_utf8_work_bytes(flat.size, n, ctypes.byref(need)))
    work = torch.empty(need.value, dtype=torch.uint8, device="cuda:0")
    info = torch.empty(5, dtype=torch.int64, device="cuda:0")
    s = torch.cuda.current_stream().cuda_stream
    batch = (0, t.data_ptr() if flat.size else None, flat.size, None if d_off is None else d_off.data_ptr(), n, stride)
    N.check(lib.acb_utf8_decode_device(*batch, errors, work.data_ptr(), need.value, info.data_ptr(), s))
    inf = info.tolist()
    out = torch.empty(max(inf[0] * width, 16), dtype=torch.uint8, device="cuda:0")
    oo = torch.empty(n + 1, dtype=torch.int64, device="cuda:0")
    N.check(lib.acb_utf8_write_device(*batch, work.data_ptr(), need.value, width, out.data_ptr(), oo.data_ptr(), s))
    o, v = oo.cpu().numpy(), out.cpu().numpy()
    dt = np.uint8 if width == 1 else "<u4"
    return [v[o[i]:o[i + 1]].view(dt).tolist() for i in range(n)], inf


def want_info(hays):
    lets = [eu.letters(h) for h in hays]
    flat_start = np.cumsum([0] + [len(h) for h in hays])
    err = [-1, -1]
    for i, h in enumerate(hays):
        e = eu.first_error(h)
        if e:
            err = [int(flat_start[i]) + e[0], int(flat_start[i]) + e[1]]
            break
    return lets, [sum(map(len, lets)), max([max(x) for x in lets if x] or [0]), max(map(len, lets), default=0)] + err


def check_c(hays, widths=(4, 1)):
    lets, info = want_info(hays)
    for w in widths:
        if w == 1 and info[1] >= 256:
            continue
        got, inf = c_decode(hays, errors=N.UTF8_STRICT, width=w)
        assert got == lets
        assert inf == info
    got, inf = c_decode(hays, errors=N.UTF8_REPLACE)
    assert inf == info[:3] + [-1, -1]


def every_code_point():
    cps = [c for c in range(0x110000) if not 0xD800 <= c <= 0xDFFF]
    return ["".join(map(chr, cps[i:i + 997])).encode() for i in range(0, len(cps), 997)]


@pytest.mark.gpu
def test_c_every_code_point():
    hays = every_code_point()
    check_c(hays)
    check_c([bytes(range(128))] * 3 + ["é".encode(), b""])          # narrow


@pytest.mark.gpu
def test_c_invalid_sequences():
    bad = [b"\xc0\xaf", b"\xe0\x80\xaf", b"\xf0\x80\x80\xaf", b"\xed\xa0\x80", b"\xed\xbf\xbf", b"\xf4\x90\x80\x80",
           b"\xf5\x80", b"\xff", b"\x80", b"\xbf\xbf\xbf\xbf", b"\xe2\x82", b"\xf0\x9f\x98", b"a\xe2", b"\xc2"]
    check_c(bad)
    # a lead at a haystack's end never takes the continuations that open the next one
    check_c([b"x\xe2", b"\x82\xacy", b"\xf0\x9f", b"\x98\x80", b"", b"\xc3", b"\xa9"])
    rng = random.Random(5)
    check_c([bytes(rng.choice(TRAPS) for _ in range(rng.randint(0, 40))) for _ in range(3000)])


@pytest.mark.gpu
def test_c_straddles_groups_and_tiles():
    rng = random.Random(7)
    letters = ["a", "é", "€", "😀", "\x00"]
    hays = []
    for n in (0, 1, 31, 32, 33, 63, 64, 65, 8191, 8192, 8193, 3 * 8192 + 5):
        s = "".join(rng.choice(letters) for _ in range(n))
        hays.append(s.encode()[:n])                                 # cut anywhere: truncated letters included
    check_c(hays)
    check_c([s.encode() for s in ("€" * 3000, "😀" * 2049, "é" * 4097 + "\xff")])   # letters across group and tile edges
    check_c([b""] * 3000 + [b"\xe2\x82\xac" * 5] + [b""] * 2000)    # many empty haystacks around one tile


@pytest.mark.gpu
def test_c_stride_rows():
    rows = np.zeros((5, 40), dtype=np.uint8)
    for i, s in enumerate([b"abc", "é€😀".encode(), b"\xe2\x82", b"", b"\xff" * 40]):
        rows[i, :len(s)] = np.frombuffer(s, dtype=np.uint8)
    hays = [bytes(r) for r in rows]
    lets, info = want_info(hays)
    for w in (4,):
        got, inf = c_decode(rows=rows, errors=N.UTF8_STRICT, width=w)
        assert got == lets and inf == info


@pytest.mark.gpu
def test_c_encode_round_trip():
    torch = _torch()
    lib = N.lib()
    for width, texts in ((4, ["".join(map(chr, range(i, min(i + 5000, 0x110000)))) for i in range(0, 0x110000, 5000)]),
                         (1, ["".join(map(chr, range(256))), "", "abc"])):
        letters = [np.frombuffer(s.encode("utf-32-le", "surrogatepass"), "<u4").astype(np.uint8 if width == 1 else "<u4")
                   for s in texts]
        flat = np.concatenate([x.view(np.uint8) for x in letters])
        offs = np.zeros(len(texts) + 1, dtype=np.int64)
        np.cumsum([x.nbytes for x in letters], out=offs[1:])
        t, d_off = torch.from_numpy(flat).cuda(), torch.from_numpy(offs).cuda()
        need = ctypes.c_int64(0)
        N.check(lib.acb_utf8_work_bytes(0, len(texts), ctypes.byref(need)))
        work = torch.empty(need.value, dtype=torch.uint8, device="cuda:0")
        cap = flat.size * 4
        out = torch.empty(cap, dtype=torch.uint8, device="cuda:0")
        oo = torch.empty(len(texts) + 1, dtype=torch.int64, device="cuda:0")
        tot = torch.empty(1, dtype=torch.int64, device="cuda:0")
        s = torch.cuda.current_stream().cuda_stream
        N.check(lib.acb_utf8_encode_device(0, t.data_ptr(), flat.size, d_off.data_ptr(), len(texts), width, work.data_ptr(),
                                           need.value, out.data_ptr(), cap, oo.data_ptr(), tot.data_ptr(), s))
        o, v = oo.cpu().numpy(), out.cpu().numpy()
        want = [x.encode("utf-8", "surrogatepass") for x in texts]
        assert [bytes(v[o[i]:o[i + 1]]) for i in range(len(texts))] == want
        assert int(tot.item()) == sum(map(len, want))


@pytest.mark.gpu
def test_c_einval():
    torch = _torch()
    lib = N.lib()
    t = torch.zeros(64, dtype=torch.uint8, device="cuda:0")
    need = ctypes.c_int64(0)
    N.check(lib.acb_utf8_work_bytes(64, 1, ctypes.byref(need)))
    work = torch.empty(need.value, dtype=torch.uint8, device="cuda:0")
    info = torch.empty(5, dtype=torch.int64, device="cuda:0")
    s = torch.cuda.current_stream().cuda_stream
    ok = (0, t.data_ptr(), 64, None, 1, 64)
    assert lib.acb_utf8_decode_device(*ok, 2, work.data_ptr(), need.value, info.data_ptr(), s) == N.ACB_EINVAL
    assert lib.acb_utf8_decode_device(*ok, 0, work.data_ptr(), need.value, None, s) == N.ACB_EINVAL
    assert lib.acb_utf8_decode_device(*ok, 0, work.data_ptr(), need.value - 1, info.data_ptr(), s) == N.ACB_EINVAL
    assert lib.acb_utf8_decode_device(0, None, 64, None, 1, 64, 0, work.data_ptr(), need.value, info.data_ptr(), s) == N.ACB_EINVAL
    assert lib.acb_utf8_decode_device(0, t.data_ptr() + 1, 63, None, 1, 63, 0, work.data_ptr(), need.value, info.data_ptr(), s) == N.ACB_EINVAL
    assert lib.acb_utf8_decode_device(0, t.data_ptr(), 64, None, 3, 64, 0, work.data_ptr(), need.value, info.data_ptr(), s) == N.ACB_EINVAL
    N.check(lib.acb_utf8_decode_device(*ok, 0, work.data_ptr(), need.value, info.data_ptr(), s))
    out = torch.empty(256, dtype=torch.uint8, device="cuda:0")
    oo = torch.empty(2, dtype=torch.int64, device="cuda:0")
    for width in (0, 2, 3, 8):
        assert lib.acb_utf8_write_device(*ok, work.data_ptr(), need.value, width, out.data_ptr(), oo.data_ptr(), s) == N.ACB_EINVAL
    assert lib.acb_utf8_write_device(*ok, work.data_ptr(), need.value, 4, None, oo.data_ptr(), s) == N.ACB_EINVAL
    assert lib.acb_utf8_write_device(*ok, work.data_ptr(), need.value, 4, out.data_ptr(), None, s) == N.ACB_EINVAL
    off = torch.tensor([0, 64], dtype=torch.int64, device="cuda:0")
    tot = torch.empty(1, dtype=torch.int64, device="cuda:0")
    enc = (0, t.data_ptr(), 64, off.data_ptr(), 1)
    assert lib.acb_utf8_encode_device(*enc, 2, work.data_ptr(), need.value, out.data_ptr(), 256, oo.data_ptr(), tot.data_ptr(), s) == N.ACB_EINVAL
    assert lib.acb_utf8_encode_device(0, t.data_ptr(), 64, None, 1, 1, work.data_ptr(), need.value, out.data_ptr(), 256, oo.data_ptr(),
                                      tot.data_ptr(), s) == N.ACB_EINVAL
    assert lib.acb_utf8_encode_device(*enc, 1, work.data_ptr(), need.value, None, 256, oo.data_ptr(), tot.data_ptr(), s) == N.ACB_EINVAL
    assert lib.acb_utf8_encode_device(*enc, 1, work.data_ptr(), need.value, out.data_ptr(), 256, oo.data_ptr(), None, s) == N.ACB_EINVAL
    assert lib.acb_utf8_work_bytes(-1, 1, ctypes.byref(need)) == N.ACB_EINVAL
    assert lib.acb_utf8_work_bytes(1, 1, None) == N.ACB_EINVAL


# ------------------------------------------------------------------------------------------------ GPU: the routes
ALPHABETS = {
    "latin1": [0x61, 0x62, 0xE9],
    "wide": [0x61, 0x142, 0x1F600],
    "mixed": [0x61, 0x62, 0x1F600],
    "fffd": [0x61, 0xFFFD, 0x41, 0x20],
}


def random_batch(rng, alphabet, invalid):
    keys = []
    for _ in range(rng.randint(2, 8)):
        k = "".join(chr(rng.choice(alphabet)) for _ in range(rng.randint(1, 4)))
        if k not in keys:
            keys.append(k)
    hays = []
    for _ in range(rng.randint(1, 12)):
        s = "".join(chr(rng.choice(alphabet + [0x20, 0x41])) for _ in range(rng.randint(0, 30)))
        raw = bytearray(s.encode())
        if invalid:
            for _ in range(rng.randint(0, 3)):
                raw.insert(rng.randint(0, len(raw)), rng.choice([0x80, 0xC3, 0xE2, 0xF0, 0xFF, 0xED]))
        hays.append(bytes(raw))
    return keys, hays


def input_forms(hays):
    """the UTF-8 input forms: list, tuple of bytearray, (flat, offsets), uint8[n, stride] and CUDA tensor (rows padded
    with NUL bytes, which decode to U+0000 and so go into the reference too)"""
    torch = _torch()
    yield "list", list(hays), hays
    yield "tuple", tuple(bytearray(h) for h in hays), hays
    flat = np.frombuffer(b"".join(hays), dtype=np.uint8)
    offs = np.zeros(len(hays) + 1, dtype=np.int64)
    np.cumsum([len(h) for h in hays], out=offs[1:])
    yield "pair", (flat, offs), hays
    width = max(map(len, hays)) or 1
    rows = np.zeros((len(hays), width), dtype=np.uint8)
    for i, h in enumerate(hays):
        rows[i, :len(h)] = np.frombuffer(h, dtype=np.uint8)
    padded = [bytes(r) for r in rows]
    yield "rows", rows, padded
    yield "cuda", torch.from_numpy(rows).cuda(), padded


def unicode_store_any(keys):
    mod = pkg.flavour("unicode")
    A = mod.Automaton(mod.STORE_ANY)
    for i, k in enumerate(keys):
        A.add_word(k, i)
    A.make_automaton()
    return A


def same(got, want, sort=True):
    g, w = triples(got), triples(want)
    assert (g if sort else sorted(g)) == (w if sort else sorted(w))


OPTION_SETS = [{}, {"whole_words": True}, {"ascii_case_insensitive": True}, {"case_insensitive": True},
               {"whole_words": True, "case_insensitive": True}]


@pytest.mark.gpu
@pytest.mark.parametrize("alphabet", sorted(ALPHABETS))
@pytest.mark.parametrize("errors", ["strict", "replace"])
def test_routes_equal_decoded_str(alphabet, errors):
    rng = random.Random(hash((alphabet, errors)) & 0xFFFF)
    for trial in range(6):
        keys, hays = random_batch(rng, ALPHABETS[alphabet], errors == "replace")
        A = unicode_store_any(keys)
        reps = {k: f"<{i}é€>" for i, k in enumerate(keys)}
        R = {"longest": A.replacer(reps), "first": A.replacer(reps, leftmost_first=True)}
        _, O = automaton("unicode", False, [[ord(c) for c in k] for k in keys])
        for form, batch, as_given in input_forms(hays):
            strs = [h.decode("utf-8", errors) for h in as_given]
            kw = dict(encoding="utf-8", errors=errors)
            for algo in ("auto", "filter", "dfa"):
                m = A.find_all_batch(batch, algo=algo, **kw)
                same(m, A.find_all_batch(strs, algo=algo))
                want = sorted(oracle_full(O, [[ord(c) for c in s] for s in strs], "wide"))
                assert sorted(zip(m.hay_id.tolist(), m.end_index.tolist(), m.values())) == want
            same(A.find_long_batch(batch, **kw), A.find_long_batch(strs))
            same(A.find_all_batch(batch, sort=False, **kw), A.find_all_batch(strs, sort=False), sort=False)
            same(A.find_all_batch(batch, ignore_white_space=True, **kw), A.find_all_batch(strs, ignore_white_space=True))
            for opts in OPTION_SETS:
                same(A.find_all_batch(batch, **opts, **kw), A.find_all_batch(strs, **opts))
                same(A.find_leftmost_longest_batch(batch, **opts, **kw), A.find_leftmost_longest_batch(strs, **opts))
                same(A.find_leftmost_first_batch(batch, **opts, **kw), A.find_leftmost_first_batch(strs, **opts))
                for r in R.values():
                    got = r.replace_batch(batch, **opts, **kw)
                    want = [s.encode("utf-8") for s in r.replace_batch(strs, **opts)]
                    if form in ("list", "tuple"):
                        assert got == want
                    else:
                        flat, offs = got
                        if form == "cuda":
                            assert flat.is_cuda and offs.is_cuda
                            flat, offs = flat.cpu().numpy(), offs.cpu().numpy()
                        assert [bytes(flat[offs[i]:offs[i + 1]]) for i in range(len(want))] == want


@pytest.mark.gpu
def test_strict_errors_match_cpython():
    A = unicode_store_any(["ab", "é", "€"])
    R = A.replacer({"ab": "x", "é": "y", "€": "z"})
    hays = [b"ab", "é€".encode(), b"x\xe2\x82", b"\xff", b"ok\xed\xa0\x80"]
    for form, batch, as_given in input_forms(hays):
        first = next(h for h in as_given if cpython(h)[1] is not None)
        try:
            first.decode("utf-8")
        except UnicodeDecodeError as e:
            want = e
        with pytest.raises(UnicodeDecodeError) as ei:
            A.find_all_batch(batch, encoding="utf-8")
        got = ei.value
        assert (got.encoding, got.object, got.start, got.end) == ("utf-8", want.object, want.start, want.end), form
        assert got.reason == want.reason
        with pytest.raises(UnicodeDecodeError):
            R.replace_batch(batch, encoding="utf-8")


@pytest.mark.gpu
def test_unencodable_replacement():
    A = unicode_store_any(["ab"])
    R = A.replacer({"ab": "x\ud800"})
    with pytest.raises(UnicodeEncodeError):
        R.replace_batch([b"zab"], encoding="utf-8")


@pytest.mark.gpu
def test_width_choice_and_launches():
    keys = ["ab", "é", "b€", "😀"]
    A = unicode_store_any(keys)
    narrow = [b"xxab", "café ab".encode(), b""]
    wide = narrow + ["b€😀".encode()]
    for hays in (narrow, wide):
        strs = [h.decode() for h in hays]
        same(A.find_all_batch(hays, encoding="utf-8"), A.find_all_batch(strs))
        b = A._utf8_batch(hays, N.UTF8_STRICT, 0)
        assert b.narrow == (hays is narrow)
    b = A._utf8_batch(narrow, N.UTF8_STRICT, 0, narrow_ok=False)
    assert not b.narrow
    # the UTF-8 route launches the decoded text's device route, a UTF-32 CUDA tensor, plus the decode
    torch = _torch()
    lib = N.lib()
    strs = ["ab€😀", "éxab", "b€ab"]                                  # 4 letters each: rows of a UTF-32 tensor
    t32 = torch.from_numpy(np.frombuffer("".join(strs).encode("utf-32-le"), np.uint8).reshape(3, 16).copy()).cuda()
    for algo in ("filter", "dfa"):
        for kw in ({}, {"whole_words": True}):
            before = lib.acb_launch_count()
            want = A.find_all_batch(t32, algo=algo, **kw)
            scan = lib.acb_launch_count() - before
            before = lib.acb_launch_count()
            same(A.find_all_batch([s.encode() for s in strs], algo=algo, encoding="utf-8", **kw), want)
            assert lib.acb_launch_count() - before == scan + DECODE_LAUNCHES


@pytest.mark.gpu
def test_past_2_gib():
    """a find_all over a CUDA UTF-8 tensor whose 4-byte letters pass 2 GiB: ~600 MB of ASCII and one 3-byte letter"""
    torch = _torch()
    n, stride = 2400, 256 * 1024                                      # 629 MB of text, 2.5 GB decoded
    A = unicode_automaton(["needle", "€x"])
    t = torch.full((n, stride), ord("a"), dtype=torch.uint8, device="cuda:0")
    plants = [(0, 10), (n // 2, 77), (n - 1, stride - 6)]
    for h, e in plants:
        t[h, e:e + 6] = torch.tensor(list(b"needle"), dtype=torch.uint8)
    t[n - 2, 100:104] = torch.tensor(list("€x".encode()), dtype=torch.uint8)   # row n-2 holds 2 letters fewer
    m = A.find_all_batch(t, encoding="utf-8")
    want = sorted([(h, e + 5, 0) for h, e in plants] + [(n - 2, 101, 1)])
    assert triples(m) == want
    del t
    torch.cuda.empty_cache()
