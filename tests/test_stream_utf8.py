"""UTF-8 stream batches (encoding="utf-8" on the stream factories): each stream holds back the bytes of an unfinished
letter on the GPU, and every feed reports what the stream batch of `str` reports when each chunk is replaced by what
CPython's incremental decoder of that stream returns for it.  CPU half: the hold rule (emul_stream_utf8) against the
decoder and the refusals.  GPU half: the C entries, every stream form and input form under both errors values against
the `str` batches fed by incremental decoders and against the whole-batch methods, strict errors, overflow retries,
finish, reset, launch counts, positions past 2^31 and a second thread."""
import codecs
import ctypes
import itertools
import random
import threading

import numpy as np
import pytest

import emul_stream_utf8 as es
import emul_utf8 as eu
import pyahocorasick_b200 as pkg
from batch_cases import triples
from pyahocorasick_b200 import _native as N
from test_utf8_batch import DECODE_LAUNCHES, TRAPS

# the launches a UTF-8 feed adds to the feed of its decoded letters: the stage (lengths, gather tiles, gather), the
# decode and the carry commit; a replacing feed adds the encode's two more
STAGE_LAUNCHES = 3 + DECODE_LAUNCHES + 1


def decoder(errors="replace"):
    return codecs.getincrementaldecoder("utf-8")(errors)


def cpython_hold(x: bytes) -> int:
    d = decoder()
    d.decode(x)
    return len(d.getstate()[0])


# ------------------------------------------------------------------------------------------------ CPU: the hold rule
def test_hold_two_bytes():
    for a in range(256):
        for b in range(256):
            x = bytes([a, b])
            assert es.hold(x) == cpython_hold(x), x


def test_hold_trap_strings():
    for k in range(5):
        for t in itertools.product(TRAPS, repeat=k):
            x = bytes(t)
            assert es.hold(x) == cpython_hold(x), x


def split_fuzz(rng):
    """a byte string of valid letters, trap bytes and truncated letters, cut at random points"""
    raw = bytearray()
    for _ in range(rng.randint(0, 12)):
        r = rng.random()
        if r < 0.5:
            raw += chr(rng.choice([0x41, 0xE9, 0x20AC, 0x2019, 0xFFFD, 0x1F600, 0x10FFFF])).encode()
        elif r < 0.8:
            raw.append(rng.choice(TRAPS))
        else:
            raw += chr(rng.choice([0xE9, 0x20AC, 0x1F600])).encode()[:rng.randint(1, 3)]
    cuts = sorted(rng.randint(0, len(raw)) for _ in range(rng.randint(0, 4)))
    return [bytes(raw[a:b]) for a, b in zip([0] + cuts, cuts + [len(raw)])]


def test_staged_decode_equals_incremental_decoder():
    rng = random.Random(421)
    for _ in range(20000):
        chunks = split_fuzz(rng)
        rep, strict, carry = decoder("replace"), decoder("strict"), b""
        broken = False
        for i, c in enumerate(chunks + [None]):
            final = c is None
            staged, new = es.stage(carry, b"" if final else c, final)
            assert eu.decode(staged) == rep.decode(b"" if final else c, final)
            assert len(new) == len(rep.getstate()[0])
            if not broken:
                err = eu.first_error(staged)
                try:
                    got = strict.decode(b"" if final else c, final)
                    assert err is None and got == eu.decode(staged)
                except UnicodeDecodeError as e:
                    assert (e.object, e.start, e.end) == (carry + (b"" if final else c), *err)
                    broken = True
            carry = new


def unicode_store_any(keys):
    mod = pkg.flavour("unicode")
    A = mod.Automaton(mod.STORE_ANY)
    for i, k in enumerate(keys):
        A.add_word(k, i)
    A.make_automaton()
    return A


def test_refusals():
    A = unicode_store_any(["ab", "é"])
    R = A.replacer({"ab": "x", "é": "y"})
    factories = [A.stream_batch, A.ascii_case_insensitive_stream_batch, A.case_insensitive_stream_batch,
                 R.stream_batch, R.ascii_case_insensitive_stream_batch, R.case_insensitive_stream_batch]
    for make in factories:
        for enc in ("latin-1", "utf-16", "no-such-codec"):
            with pytest.raises(ValueError):
                make(2, encoding=enc)
        with pytest.raises(ValueError):
            make(2, encoding="utf-8", errors="ignore")
        with pytest.raises(ValueError):
            make(2, errors="replace")                                 # errors without an encoding
    with pytest.raises(ValueError):                                   # what the str batches refuse stays refused
        A.stream_batch(2, long=True, whole_words=True, encoding="utf-8")
    with pytest.raises(UnicodeEncodeError):
        A.replacer({"ab": "x\ud800", "é": "y"}).stream_batch(2, encoding="utf-8")
    B = pkg.flavour("bytes").Automaton(pkg.STORE_INTS)
    B.add_word(b"ab", 0)
    B.make_automaton()
    with pytest.raises(ValueError):
        B.stream_batch(2, encoding="utf-8")
    mod = pkg.flavour("unicode")
    S = mod.Automaton(mod.STORE_INTS, mod.KEY_SEQUENCE)
    S.add_word((1, 2), 0)
    S.make_automaton()
    with pytest.raises(ValueError):
        S.stream_batch(2, encoding="utf-8")


# ------------------------------------------------------------------------------------------------ GPU: the C entries
def _torch():
    import torch
    return torch


class Carry:
    """acb_utf8_carry_* on cuda:0"""

    def __init__(self, n):
        self.lib = N.lib()
        self.h = ctypes.c_void_p()
        N.check(self.lib.acb_utf8_carry_new(0, n, ctypes.byref(self.h)))
        self.n = n

    def __del__(self):
        self.lib.acb_utf8_carry_free(self.h)

    def stage(self, chunks, ids=None, final=False, commit=True):
        """the staged haystacks of a feed of byte chunks (as a ragged CUDA batch), committed unless told otherwise"""
        torch = _torch()
        flat = np.frombuffer(b"".join(chunks) + b"\0", dtype=np.uint8)[:-1]
        offs = np.zeros(len(chunks) + 1, dtype=np.int64)
        np.cumsum([len(c) for c in chunks], out=offs[1:])
        n, total = len(chunks), int(flat.size)
        t = torch.from_numpy(flat.copy()).cuda() if total else None
        d_offs = torch.from_numpy(offs).cuda()
        d_ids = None if ids is None else torch.tensor(ids, dtype=torch.int32, device="cuda")
        span = total + 3 * n
        staged = torch.full((span + 16,), 0xAB, dtype=torch.uint8, device="cuda")
        soffs = torch.empty(n + 1, dtype=torch.int64, device="cuda")
        stream = torch.cuda.current_stream().cuda_stream
        N.check(self.lib.acb_utf8_carry_stage_device(self.h, None if t is None else t.data_ptr(), total, d_offs.data_ptr(), n, 0,
                                                     None if d_ids is None else d_ids.data_ptr(), int(final), staged.data_ptr(),
                                                     span, soffs.data_ptr(), stream))
        if commit:
            N.check(self.lib.acb_utf8_carry_commit_device(self.h, None if d_ids is None else d_ids.data_ptr(), n, stream))
        s, o = staged.cpu().numpy(), soffs.cpu().numpy()
        assert not s[o[-1]:span].any() and (s[span:] == 0xAB).all()   # zeros up to the span, nothing past it
        return [bytes(s[o[h]:o[h + 1]]) for h in range(n)]

    def pending(self):
        out = np.zeros(max(self.n, 1), dtype=np.int64)
        N.check(self.lib.acb_utf8_carry_pending(self.h, N.ptr(out), len(out)))
        return out[:self.n].tolist()

    def held(self, s):
        b, k = (ctypes.c_uint8 * 3)(), ctypes.c_int32(0)
        N.check(self.lib.acb_utf8_carry_bytes(self.h, s, b, ctypes.byref(k)))
        return bytes(b)[:k.value]


class Model:
    """emul_stream_utf8 per stream"""

    def __init__(self, n):
        self.carry = [b""] * n

    def stage(self, chunks, ids=None, final=False):
        out = []
        for h, c in enumerate(chunks):
            s = h if ids is None else ids[h]
            staged, self.carry[s] = es.stage(self.carry[s], c, final)
            out.append(staged)
        return out


LETTERS = ["A", "é", "€", "😀", "�", "\U0010FFFF"]


@pytest.mark.gpu
def test_c_stage_and_commit():
    cases = []
    for a, b in itertools.product(LETTERS, repeat=2):                 # every split point of every 1- to 4-byte letter
        x = (a + b).encode()
        cases.append([[x[:i]] for i in range(len(x) + 1)] + [[x[i:]] for i in range(len(x) + 1)])
    cases.append([[bytes([0xF0])], [bytes([0x9F])], [bytes([0x98])], [bytes([0x80])]])   # a carry grows to 3 bytes
    cases.append([[b"", b"x\xe2"], [b"\x82", b""], [b"", b"\xac"], [b"\xac", b""]])       # empty chunks
    cases.append([[b"\xe0", b"\xed", b"\xf0", b"\xf4", b"\xc2"], [b"\x80", b"\xa0", b"\x8f", b"\x90", b"A"]])   # straddles
    for feeds in cases:
        n = max(len(f) for f in feeds)
        C, M = Carry(n), Model(n)
        for f in feeds:
            assert C.stage(f) == M.stage(f)
            assert C.pending() == [len(c) for c in M.carry]
            assert [C.held(s) for s in range(n)] == M.carry
        assert C.stage([b""] * n, final=True) == M.stage([b""] * n, final=True)
        assert C.pending() == [0] * n
    rng = random.Random(7)
    C, M = Carry(9), Model(9)
    for _ in range(60):                                               # ids in any order, some streams left out
        ids = rng.sample(range(9), rng.randint(0, 9))
        chunks = [b"".join(split_fuzz(rng))[:rng.randint(0, 6)] for _ in ids]
        final = rng.random() < 0.1
        assert C.stage(chunks, ids, final) == M.stage(chunks, ids, final)
        assert [C.held(s) for s in range(9)] == M.carry
    before = C.pending()                                              # a stage without a commit changes nothing ...
    staged = C.stage([b"\xf0\x9f"] * 9, commit=False)
    assert C.pending() == before
    assert C.stage([b"\xf0\x9f"] * 9) == staged                       # ... and the next stage restages from the carry
    N.check(C.lib.acb_utf8_carry_reset(C.h, N.ptr(np.array([3, 5], np.int32)), 2))
    assert [p for s, p in enumerate(C.pending()) if s in (3, 5)] == [0, 0]


@pytest.mark.gpu
def test_c_einval():
    torch = _torch()
    C = Carry(4)
    lib, s = C.lib, torch.cuda.current_stream().cuda_stream
    t = torch.zeros(64, dtype=torch.uint8, device="cuda")
    o = torch.zeros(5, dtype=torch.int64, device="cuda")
    st = torch.zeros(128, dtype=torch.uint8, device="cuda")
    ok = (C.h, t.data_ptr(), 16, None, 4, 4, None, 0, st.data_ptr(), 28, o.data_ptr(), s)
    N.check(lib.acb_utf8_carry_stage_device(*ok))
    for i, v in ((4, 5), (8, st.data_ptr() + 1), (9, 27), (5, 3), (1, t.data_ptr() + 4), (10, None)):
        bad = list(ok)
        bad[i] = v
        assert lib.acb_utf8_carry_stage_device(*bad) == N.ACB_EINVAL, i
    N.check(lib.acb_utf8_carry_stage_device(*ok))
    assert lib.acb_utf8_carry_commit_device(C.h, None, 3, s) == N.ACB_EINVAL     # not the staged chunk count
    N.check(lib.acb_utf8_carry_commit_device(C.h, None, 4, s))
    assert lib.acb_utf8_carry_commit_device(C.h, None, 4, s) == N.ACB_EINVAL     # nothing staged
    assert lib.acb_utf8_carry_reset(C.h, N.ptr(np.array([4], np.int32)), 1) == N.ACB_EINVAL


# ------------------------------------------------------------------------------------------------ GPU: the stream forms
KEYS = ["ab", "é", "€x", "😀", "�", "b€😀", "xx", "é€"]


def forms(chunks):
    """(form, feed argument, the bytes each chunk really holds): list, tuple of bytearray, pair, rows, CUDA tensor (rows
    padded with NUL bytes, which belong to the chunk)"""
    torch = _torch()
    yield "list", [c if c else None for c in chunks], chunks
    yield "tuple", tuple(bytearray(c) for c in chunks), chunks
    flat = np.frombuffer(b"".join(chunks) + b"\0", dtype=np.uint8)[:-1].copy()
    offs = np.zeros(len(chunks) + 1, dtype=np.int64)
    np.cumsum([len(c) for c in chunks], out=offs[1:])
    yield "pair", (flat, offs), chunks
    width = max(map(len, chunks), default=0) or 1
    rows = np.zeros((len(chunks), width), dtype=np.uint8)
    for i, c in enumerate(chunks):
        rows[i, :len(c)] = np.frombuffer(c, dtype=np.uint8)
    yield "rows", rows, [bytes(r) for r in rows]
    yield "cuda", torch.from_numpy(rows).cuda(), [bytes(r) for r in rows]


def random_feeds(rng, n_streams, invalid, equal=False):
    """feeds of (chunks, ids or None): each stream's text (valid UTF-8 unless `invalid`) cut at random bytes, so letters
    split across chunks; the last feed gives every stream the rest of its text.  equal: the chunks of a feed have one
    length (a text that runs short goes on with "x"), so rows need no NUL padding"""
    texts = []
    for _ in range(n_streams):
        raw = bytearray("".join(rng.choice("abx é€😀�") for _ in range(rng.randint(0, 24))).encode())
        if invalid:
            for _ in range(rng.randint(0, 3)):
                raw.insert(rng.randint(0, len(raw)), rng.choice([0x80, 0xC3, 0xE2, 0xF0, 0xFF, 0xED]))
        texts.append(raw)
    at, feeds = [0] * n_streams, []
    for last in [False] * rng.randint(1, 4) + [True]:
        ids = None if last or rng.random() < 0.4 else rng.sample(range(n_streams), rng.randint(1, n_streams))
        sids = range(n_streams) if ids is None else ids
        size = rng.randint(1 if equal else 0, 7)                # rows of a feed of empty chunks would hold one NUL
        if last:
            size = max(len(texts[s]) - at[s] for s in sids)
        chunks = []
        for s in sids:
            cut = at[s] + size if equal or last else min(at[s] + rng.randint(0, 7), len(texts[s]))
            if equal and cut > len(texts[s]):
                texts[s] += b"x" * (cut - len(texts[s]))
            chunks.append(bytes(texts[s][at[s]:cut]))
            at[s] = cut
        feeds.append((chunks, ids))
    return feeds


def as_texts(out):
    """a replacing feed's output as a list of bytes, whatever its form"""
    if isinstance(out, list):
        return out
    flat, offs = out
    if hasattr(flat, "is_cuda"):
        assert flat.is_cuda and offs.is_cuda
        flat, offs = flat.cpu().numpy(), offs.cpu().numpy()
    return [bytes(flat[offs[i]:offs[i + 1]]) for i in range(len(offs) - 1)]


def run(make, feeds, errors, form, replacing=False, has_finish=True):
    """feed a UTF-8 batch and the str batch of the same options (fed by one incremental decoder per stream) alike, and
    check every feed and finish; returns each stream's bytes and its matches or output over the run"""
    U, S = make(encoding="utf-8", errors=errors), make()
    assert (U.encoding, U.errors, S.encoding) == ("utf-8", errors, None)
    n = U.n_streams
    decs = [decoder(errors) for _ in range(n)]
    text = [b""] * n
    got = [[] for _ in range(n)] if not replacing else [b""] * n
    for chunks, ids in feeds:
        for f, batch, given in forms(chunks):
            if f != form:
                continue
            sids = range(len(given)) if ids is None else ids
            strs = [decs[s].decode(c) for s, c in zip(sids, given)]
            for s, c in zip(sids, given):
                text[s] += c
            out, want = U.feed(batch, ids), S.feed(strs, ids)
            if replacing:
                out = as_texts(out)
                assert out == [w.encode() for w in want]
                for s, o in zip(sids, out):
                    got[s] += o
            else:
                assert triples(out) == triples(want)
                for s, e, k in triples(out):
                    got[s].append((e, k))
            assert (U.positions == S.positions).all()
            assert U.pending.tolist() == [len(d.getstate()[0]) for d in decs]
    if has_finish:
        tails = [d.decode(b"", True) for d in decs]
        out = U.finish()
        if replacing:
            want = [a.encode() + b.encode() for a, b in zip(S.feed(tails), S.finish())]
            assert out == want
            got = [g + o for g, o in zip(got, out)]
        else:
            want = triples(S.feed(tails))
            if S.leftmost_longest or S.leftmost_first or S.whole_words:
                # one final feed against a feed and a finish: the same records of each stream, in the same order
                want = sorted(want + triples(S.finish()), key=lambda r: r[0])
            assert triples(out) == want
            for s, e, k in triples(out):
                got[s].append((e, k))
        assert (U.positions == 0).all() and (U.pending == 0).all()
    return text, got


STREAM_FORMS = {
    "find_all": lambda A, R: (lambda **kw: A.stream_batch(5, **kw)),
    "find_all_dfa": lambda A, R: (lambda **kw: A.stream_batch(5, algo="dfa", **kw)),
    "long": lambda A, R: (lambda **kw: A.stream_batch(5, long=True, **kw)),
    "white_space": lambda A, R: (lambda **kw: A.stream_batch(5, ignore_white_space=True, **kw)),
    "leftmost_longest": lambda A, R: (lambda **kw: A.stream_batch(5, leftmost_longest=True, **kw)),
    "leftmost_first": lambda A, R: (lambda **kw: A.stream_batch(5, leftmost_first=True, **kw)),
    "words": lambda A, R: (lambda **kw: A.stream_batch(5, whole_words=True, **kw)),
    "words_leftmost": lambda A, R: (lambda **kw: A.stream_batch(5, whole_words=True, leftmost_longest=True, **kw)),
    "ascii_fold": lambda A, R: (lambda **kw: A.ascii_case_insensitive_stream_batch(5, **kw)),
    "unicode_fold": lambda A, R: (lambda **kw: A.case_insensitive_stream_batch(5, leftmost_first=True, **kw)),
    "replace": lambda A, R: (lambda **kw: R.stream_batch(5, **kw)),
    "replace_ascii_fold": lambda A, R: (lambda **kw: R.ascii_case_insensitive_stream_batch(5, whole_words=True, **kw)),
    "replace_unicode_fold": lambda A, R: (lambda **kw: R.case_insensitive_stream_batch(5, **kw)),
}


@pytest.mark.gpu
@pytest.mark.parametrize("errors", ["strict", "replace"])
@pytest.mark.parametrize("form", ["list", "tuple", "pair", "rows", "cuda"])
def test_every_stream_form(form, errors):
    A = unicode_store_any(KEYS)
    R = A.replacer({k: f"<{i}é😀>" for i, k in enumerate(KEYS)})
    rng = random.Random(f"{form} {errors}")
    for name, mk in STREAM_FORMS.items():
        for _ in range(3):
            feeds = random_feeds(rng, 5, errors == "replace", form in ("rows", "cuda"))
            replacing = name.startswith("replace")
            text, got = run(mk(A, R), feeds, errors, form, replacing)
            if name in ("find_all", "leftmost_longest", "replace"):
                # over all feeds and finish: the whole-batch method on each stream's concatenated bytes
                if name == "find_all":
                    want = A.find_all_batch(text, encoding="utf-8", errors=errors)
                elif name == "leftmost_longest":
                    want = A.find_leftmost_longest_batch(text, encoding="utf-8", errors=errors)
                if replacing:
                    assert got == R.replace_batch(text, encoding="utf-8", errors=errors)
                else:
                    assert sorted((s, e, k) for s in range(5) for e, k in got[s]) == sorted(triples(want))


@pytest.mark.gpu
@pytest.mark.parametrize("errors", ["strict", "replace"])
def test_invalid_sequences_straddling_chunks(errors):
    A = unicode_store_any(KEYS)
    R = A.replacer({k: "#" for k in KEYS})
    pairs = [(b"\xe0", b"\x80"), (b"\xed", b"\xa0"), (b"\xf0", b"\x8f"), (b"\xf4", b"\x90"), (b"\xc2", b"\x41"),
             (b"\xe2\x82", b"\xac\x80"), (b"\xf0\x9f", b"A")]
    makers = [(lambda **kw: A.stream_batch(2, **kw), False),
              (lambda **kw: A.stream_batch(2, leftmost_longest=True, **kw), False),
              (lambda **kw: R.stream_batch(2, **kw), True)]
    for a, b in pairs:
        # the second chunk of stream 1 is a stray continuation byte after a completed carry
        feeds = [([a, b"ab\xe2\x82"], None), ([b, b"\xac\x80"], None), ([b"\xbf", b""], None)]
        for make, replacing in makers:
            if errors == "replace":
                run(make, feeds, errors, "list", replacing)
                continue
            U, decs = make(encoding="utf-8"), [decoder("strict") for _ in range(2)]
            for chunks, _ in feeds:
                want = None
                for d, c in zip(decs, chunks):
                    try:
                        d.decode(c)
                    except UnicodeDecodeError as e:
                        want = (e.encoding, e.object, e.start, e.end, e.reason)
                        break
                if want is None:
                    U.feed(chunks)
                    continue
                assert raised(lambda: U.feed(chunks)) == want
                break


def raised(call):
    with pytest.raises(UnicodeDecodeError) as ei:
        call()
    e = ei.value
    return e.encoding, e.object, e.start, e.end, e.reason


@pytest.mark.gpu
def test_strict_errors():
    A = unicode_store_any(KEYS)
    R = A.replacer({k: "#" for k in KEYS})
    for make in (lambda: A.stream_batch(3, encoding="utf-8"), lambda: A.stream_batch(3, whole_words=True, encoding="utf-8"),
                 lambda: R.stream_batch(3, encoding="utf-8")):
        for form in ("list", "pair", "rows", "cuda"):
            U = make()
            decs = [decoder("strict") for _ in range(3)]
            first = [b"ab\xf0\x9f", b"xyz\xe2", b"abc\xc3"]             # one length: rows need no padding
            for f, batch, given in forms(first):
                if f == form:
                    U.feed(batch)
                    for d, c in zip(decs, given):
                        d.decode(c)
            pos, pend = U.positions, U.pending
            bad = [b"\x98\x80", b"\x82A", b"\xff"]                     # chunk 1 is the first invalid one
            for f, batch, given in forms(bad):
                if f != form:
                    continue
                want = raised(lambda: decs[1].decode(given[1]))
                got = raised(lambda: U.feed(batch))
                assert got == want
            assert (U.positions == pos).all() and (U.pending == pend).all()
            U.feed([b"\x98\x80", b"\x82\xacab", b"\xa9"])               # the feed that raised left every carry
            assert U.positions.tolist() == [pos[0] + 1, pos[1] + 3, pos[2] + 1]
            U.feed([b"", b"", b"\xe2\x82"])
            pos = U.positions
            d = decoder("strict")
            d.decode(b"\xe2\x82")
            assert raised(lambda: U.finish([2])) == raised(lambda: d.decode(b"", True))
            assert (U.positions == pos).all()
            assert U.pending.tolist() == [0, 0, 2]


@pytest.mark.gpu
def test_overflow_retry_commits_once():
    A = unicode_store_any(["a", "é"])
    U = A.stream_batch(2, encoding="utf-8")
    S = A.stream_batch(2)
    A._match_cap = 0
    chunks = [b"a" * 6000 + b"\xc3", b"\xc3"]
    m = U.feed(chunks)
    assert triples(m) == triples(S.feed(["a" * 6000, ""]))
    assert U.pending.tolist() == [1, 1]
    m = U.feed([b"\xa9", b"\xa9a"])
    assert triples(m) == triples(S.feed(["é", "éa"]))
    assert U.positions.tolist() == [6001, 2]


@pytest.mark.gpu
def test_finish_and_reset():
    A = unicode_store_any(KEYS)
    S = A.stream_batch(2)
    with pytest.raises(ValueError):
        S.finish()                                                    # a find_all batch of letters has none
    for kw in ({}, {"long": True}, {"ignore_white_space": True}):
        U = A.stream_batch(2, encoding="utf-8", errors="replace", **kw)
        U.feed([b"ab \xe2\x82", b"x"])
        assert U.pending.tolist() == [2, 0]
        m = U.finish([0])
        assert triples(m) == [(0, 3, KEYS.index("�"))]
        assert U.positions.tolist() == [0, 1] and U.pending.tolist() == [0, 0]
        U.feed([b"\xf0\x9f", b"\xe2"])
        U.reset([0])
        assert U.pending.tolist() == [0, 1] and U.positions.tolist() == [0, 1]
        U.reset()
        assert U.pending.tolist() == [0, 0]


@pytest.mark.gpu
def test_launch_counts():
    A = unicode_store_any(KEYS)
    R = A.replacer({k: "#" for k in KEYS})
    lib = N.lib()
    chunks = ["ab€😀", "éxab", "b€ab"]                               # 4 letters each: rows of a UTF-32 tensor
    torch = _torch()
    t32 = torch.from_numpy(np.frombuffer("".join(chunks).encode("utf-32-le"), np.uint8).reshape(3, 16).copy()).cuda()
    u8 = [c.encode() for c in chunks]
    for kw in ({}, {"leftmost_longest": True}, {"whole_words": True}):
        S, U = A.stream_batch(3, **kw), A.stream_batch(3, encoding="utf-8", **kw)
        before = lib.acb_launch_count()
        want = S.feed(t32)
        plain = lib.acb_launch_count() - before
        before = lib.acb_launch_count()
        assert triples(U.feed(u8)) == triples(want)
        assert lib.acb_launch_count() - before == plain + STAGE_LAUNCHES
    S, U = R.stream_batch(3), R.stream_batch(3, encoding="utf-8")
    before = lib.acb_launch_count()
    S.feed(t32)
    plain = lib.acb_launch_count() - before
    before = lib.acb_launch_count()
    U.feed(u8)
    assert lib.acb_launch_count() - before == plain + STAGE_LAUNCHES + 2


@pytest.mark.gpu
def test_position_past_2_31():
    torch = _torch()
    A = unicode_store_any(["x😀", "😀ab"])
    U = A.stream_batch(1, encoding="utf-8")
    half = 1 << 30
    c1 = torch.full((1, half), ord("x"), dtype=torch.uint8, device="cuda")
    assert U.feed(c1).end_index.size == 0
    del c1
    c2 = torch.full((1, half), ord("x"), dtype=torch.uint8, device="cuda")
    c2[0, -2:] = torch.tensor([0xF0, 0x9F], dtype=torch.uint8)
    assert U.feed(c2).end_index.size == 0
    del c2
    assert U.positions.tolist() == [2 * half - 2] and U.pending.tolist() == [2]
    m = U.feed([b"\x98\x80ab"])
    assert list(zip(m.end_index.tolist(), m.key_id.tolist())) == [(2 * half - 2, 0), (2 * half, 1)]
    assert m.end_index.dtype == np.int64


@pytest.mark.gpu
def test_second_thread():
    A = unicode_store_any(KEYS)
    rng = random.Random(5)
    runs = [random_feeds(rng, 5, True) for _ in range(2)]
    errs = []

    def work(feeds):
        try:
            for _ in range(4):
                run(lambda **kw: A.stream_batch(5, leftmost_longest=True, **kw), feeds, "replace", "list")
        except Exception as e:                                        # noqa: BLE001 -- reported below
            errs.append(e)
    th = threading.Thread(target=work, args=(runs[1],))
    th.start()
    work(runs[0])
    th.join()
    assert not errs, errs
