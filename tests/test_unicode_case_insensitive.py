"""case_insensitive=True of find_all_batch, find_leftmost_longest_batch, find_leftmost_first_batch and
Replacer.replace_batch: keys and text compared under Unicode simple case folding (each class of letters folded to its
lowest code point), the text folded on the GPU by a table-driven kernel, the word test and the rewrite on the text as
given.

The CPU half checks the restatement (tests/emul_unicode_fold.py) against Python's `re` with IGNORECASE, the map, the key
groups the Automaton builds and the refusals; the gpu-marked half runs every code point through the device fold and the
real routes against the restatement, against the ASCII fold on ASCII text, and past 2 GiB."""
import ctypes
import re

import numpy as np
import pytest

import emul_unicode_fold as eu
import pyahocorasick_b200 as pkg
from batch_cases import forms, triples
from pyahocorasick_b200 import _native as N
from pyahocorasick_b200.automaton import _FOLD_UNICODE, _unicode_fold_map

# letters that fold in more than pairs, fold across latin-1, or look alike and must not fold; ı (U+0131) is left out:
# `re` matches it with I, simple folding does not (pinned in test_what_does_not_fold)
TRAPS = [0x4B, 0x6B, 0x212A, 0x53, 0x73, 0x17F, 0xB5, 0x39C, 0x3BC, 0x3A3, 0x3C3, 0x3C2, 0xC9, 0xE9, 0x178, 0xFF,
         0xDF, 0x1E9E, 0x1C5, 0x1C4, 0x1C6, 0x10400, 0x10428, 0x13A0, 0xAB70, 0x10D0, 0x1C90, 0x61, 0x41]
LATIN1 = [c for c in TRAPS if c < 256] + [0xC0, 0xE0, 0xD7, 0xF7]


def text(letters):
    return "".join(map(chr, letters))


def random_case(rng, alphabet, n_keys=None, n_hays=None):
    keys = []
    for _ in range(n_keys or int(rng.integers(1, 9))):
        k = [int(x) for x in rng.choice(alphabet, size=int(rng.integers(1, 5)))]
        if k not in keys:
            keys.append(k)
        if rng.integers(0, 3) == 0:                              # a case variant of it
            v = [ord(chr(x).swapcase()) if len(chr(x).swapcase()) == 1 else x for x in k]
            if v not in keys:
                keys.append(v)
    hays = [[int(x) for x in rng.choice(alphabet, size=int(rng.integers(0, 40)))] for _ in range(n_hays or int(rng.integers(1, 6)))]
    return keys, hays


def build(keys):
    """the unicode-flavour Automaton (STORE_INTS, value = key id) over keys given as code points"""
    mod = pkg.flavour("unicode")
    A = mod.Automaton(mod.STORE_INTS)
    for i, k in enumerate(keys):
        A.add_word(text(k), i)
    A.make_automaton()
    return A


# ------------------------------------------------------------------ `re` (CPU)
def re_find_all(keys, hays):
    out = []
    for h, hay in enumerate(hays):
        for kid, k in enumerate(keys):
            for m in re.finditer("(?=" + re.escape(text(k)) + ")", text(hay), re.IGNORECASE):
                out.append((h, m.start() + len(k) - 1, -len(k), kid))
    return [(h, e, k) for h, e, _, k in sorted(out)]


def re_alternation(keys, first):
    order = sorted(range(len(keys)), key=(lambda i: i) if first else (lambda i: (-len(keys[i]), i)))
    return order, re.compile("|".join("(" + re.escape(text(keys[i])) + ")" for i in order), re.IGNORECASE)


def test_restatement_agrees_with_re():
    rng = np.random.default_rng(19)
    for _ in range(150):
        keys, hays = random_case(rng, TRAPS)
        assert eu.find_all(keys, hays) == re_find_all(keys, hays), (keys, hays)
        reps = [[0x5F] * int(rng.integers(0, 3)) + k[:1] for k in keys]
        for first in (True, False):
            order, pat = re_alternation(keys, first)
            want = [(h, m.end() - 1, order[m.lastindex - 1]) for h, hay in enumerate(hays) for m in pat.finditer(text(hay))]
            assert eu.leftmost(keys, hays, first) == want, (keys, hays, first)
            got = [text(x) for x in eu.replace(keys, reps, hays, first)]
            assert got == [pat.sub(lambda m: text(reps[order[m.lastindex - 1]]), text(hay)) for hay in hays]


def test_what_does_not_fold():
    """one letter to one letter, no Turkic rule, no normalisation"""
    def same(a, b):
        return eu.fold([ord(c) for c in a]).tolist() == eu.fold([ord(c) for c in b]).tolist()
    assert same("Müller", "MÜLLER") and same("Σοφία", "ΣΟΦΊΑ") and same("Straße", "STRAẞE") and same("Kelvin", "kELVIN")
    assert same("σ", "ς") and same("ſ", "S") and same("µ", "Μ") and same("ǅ", "ǆ") and same("\U00010400", "\U00010428")
    assert not same("ß", "s") and not same("ı", "i") and not same("İ", "i")
    assert eu.find_all([[0x73, 0x73]], [[0xDF]]) == [] and eu.find_all([[0xDF]], [[0x53, 0x53]]) == []
    assert eu.find_all([[0x66, 0x69]], [[0xFB01]]) == []                     # ﬁ is not fi
    assert eu.fold([0x390]).tolist() == [0x390]                              # ΐ stays itself
    for turkic in (0x131, 0x130):                                            # ı, İ
        assert eu.fold([turkic]).tolist() == [turkic]
        assert eu.find_all([[0x69]], [[turkic]]) == [] and eu.find_all([[0x49]], [[turkic]]) == []
    assert eu.find_all([[0x65, 0x301]], [[0xE9]]) == [] and eu.find_all([[0xE9]], [[0x65, 0x301]]) == []
    assert eu.fold([0xD800, 0xDFFF, 0x110000, 0xFFFFFFFF]).tolist() == [0xD800, 0xDFFF, 0x110000, 0xFFFFFFFF]


def test_map_properties():
    frm, to = _unicode_fold_map()
    f, t = frm.astype(np.int64), to.astype(np.int64)
    assert frm.dtype == to.dtype == np.uint32 and len(f) == len(t) > 1000
    assert np.all(np.diff(f) > 0) and np.all(t < f)
    assert not np.isin(t, f).any()                                           # idempotent: a folded letter stays
    assert np.all(t[f < 256] < 256)                                          # latin-1 closed
    assert sorted(f[(f >= 256) & (t < 256)].tolist()) == [0x178, 0x17F, 0x39C, 0x3BC, 0x1E9E, 0x212A, 0x212B]
    canon = eu.canonical()
    changed = np.flatnonzero(canon != np.arange(0x110000))
    assert np.array_equal(changed, f) and np.array_equal(canon[changed], t)
    assert not (frm.flags.writeable or to.flags.writeable)


def keys_in(A, core, narrow):
    """{folded key bytes: id} of a folded host trie, found through acb_trie_find"""
    got = {}
    fold = dict(zip(*(a.tolist() for a in _unicode_fold_map())))
    for key in A._key_objs:
        f = key.translate(fold)
        try:
            raw = f.encode("latin-1") if narrow else A._raw_key(f)[0]
        except UnicodeEncodeError:
            continue
        k, pre = ctypes.c_int32(-1), ctypes.c_int32(0)
        N.check(A._lib.acb_trie_find(core.trie, raw, len(raw), ctypes.byref(k), ctypes.byref(pre)))
        got[raw] = k.value
    assert A._lib.acb_trie_count(core.trie) == len(got)
    return got


@pytest.mark.parametrize("narrow", [False, True])
def test_folded_trie_holds_representatives(narrow):
    words = ["kelvin", "\u212Aelvin", "KELVIN", "\u00B5", "\u03BC", "\u039C", "σοφία", "ΣΟΦΊΑ", "\u017Fs", "SS",
             "\u0178", "\u00FF", "\u1E9E", "\u00DF", "x", "\u01C4", "\u01C5", "\U00010400", "\U00010428", "\u00C5",
             "\u212B", "\u0131", "\u0130", "i"]
    A = build([list(map(ord, w)) for w in words])
    core = A._fold_host(narrow, _FOLD_UNICODE)
    letters = [list(map(ord, w)) for w in words]
    live = [k if not narrow or max(eu.fold(k)) < 256 else None for k in letters]
    rep, aliases = eu.groups(live)
    got = keys_in(A, core, narrow)
    assert sorted(set(got.values())) == sorted(set(rep.values()))
    ptr = np.zeros(max(rep.values()) + 2, dtype=np.int64)
    for r, ids in aliases.items():
        ptr[r + 1] = len(ids)
    assert core.alias_ptr.tolist() == np.cumsum(ptr).tolist()
    assert core.alias_ids.tolist() == [k for r in sorted(aliases) for k in aliases[r]]
    # the non-latin-1 letters that fold into latin-1 join the 1-byte groups: Kelvin sign, μ, Μ, ſ, ẞ, Ÿ, Å-sign
    assert aliases[0] == [1, 2] and aliases[3] == [4, 5] and aliases[8] == [9] and aliases[10] == [11]
    assert aliases[12] == [13] and aliases[19] == [20]
    assert 21 not in aliases and 22 not in aliases and aliases.get(23) is None    # ı, İ and i stay apart
    if not narrow:
        assert aliases[6] == [7] and aliases[15] == [16] and aliases[17] == [18]


def test_refusals():
    A = build([[0x61, 0x62]])
    for call in (lambda: A.find_all_batch(["ab"], ignore_white_space=True, case_insensitive=True),
                 lambda: A.find_all_batch(["ab"], algo="long", case_insensitive=True),
                 lambda: A.find_long_batch(["ab"], case_insensitive=True),
                 lambda: A.find_all_batch(["ab"], ascii_case_insensitive=True, case_insensitive=True),
                 lambda: A.find_leftmost_first_batch(["ab"], ascii_case_insensitive=True, case_insensitive=True),
                 lambda: A.replacer({"ab": "x"}).replace_batch(["ab"], ascii_case_insensitive=True, case_insensitive=True)):
        with pytest.raises(ValueError):
            call()
    B = pkg.flavour("bytes").Automaton()
    B.add_word(b"ab", 0)
    B.make_automaton()
    for call in (lambda: B.find_all_batch([b"ab"], case_insensitive=True),
                 lambda: B.find_leftmost_longest_batch([b"ab"], case_insensitive=True),
                 lambda: B.find_leftmost_first_batch([b"ab"], case_insensitive=True),
                 lambda: B.replacer({b"ab": b"x"}).replace_batch([b"ab"], case_insensitive=True),
                 lambda: B.case_insensitive_stream_batch(2),
                 lambda: B.replacer({b"ab": b"x"}).case_insensitive_stream_batch(2)):
        with pytest.raises(ValueError, match="ascii_case_insensitive"):
            call()
    mod = pkg.flavour("unicode")
    S = mod.Automaton(mod.STORE_INTS, mod.KEY_SEQUENCE)
    S.add_word((1, 2), 0)
    S.make_automaton()
    for call in (lambda: S.find_all_batch([(1, 2)], case_insensitive=True),
                 lambda: S.find_leftmost_longest_batch([(1, 2)], case_insensitive=True),
                 lambda: S.case_insensitive_stream_batch(1)):
        with pytest.raises(ValueError, match="KEY_SEQUENCE"):
            call()
    import inspect
    for m in (A.stream_batch, A.ascii_case_insensitive_stream_batch, pkg.automaton.Replacer.stream_batch, A.iter,
              A.find_all, A.exists_batch):
        assert "case_insensitive" not in inspect.signature(m).parameters


# ------------------------------------------------------------------ the GPU
def wide_pair(hays):
    """(flat uint8, int64 byte offsets) of haystacks of 4-byte letters, any uint32 value"""
    offs = np.zeros(len(hays) + 1, dtype=np.int64)
    np.cumsum([4 * len(h) for h in hays], out=offs[1:])
    flat = np.concatenate([np.asarray(h, dtype="<u4") for h in hays]).view(np.uint8) if hays else np.empty(0, np.uint8)
    return flat, offs


def class_keys():
    """one single-letter key per canonical letter of every class with two or more members, and {canonical: key id}"""
    _, to = _unicode_fold_map()
    canon = sorted(set(to.tolist()))
    return [[c] for c in canon], {c: i for i, c in enumerate(canon)}


def want_single(letters, ids):
    """(end, key id) that find_all of the single-letter class keys reports in one haystack"""
    f = eu.fold(letters).tolist()
    return [(e, ids[c]) for e, c in enumerate(f) if c in ids]


@pytest.fixture
def cta_limit():
    """limit(A, n): the CTA limit of every Unicode-folded device-0 table of A (both widths); every table is set back
    to 0 after (A is kept alive until then: its tables go with it)"""
    seen = []

    def limit(A, n):
        for narrow in (False, True):
            tb = A._table_for(0, narrow, _FOLD_UNICODE)
            if tb is not None:
                N.check(N.lib().acb_table_set_cta_limit(tb, n))
                seen.append((A, tb))
    yield limit
    for _, tb in seen:
        N.check(N.lib().acb_table_set_cta_limit(tb, 0))


@pytest.mark.gpu
@pytest.mark.parametrize("limit", [1, 0])
def test_gpu_every_code_point(limit, cta_limit):
    """Every code point 0..0x10FFFF (surrogates included) and values above it, in one haystack, through the device fold
    of 4-byte letters as a CUDA tensor and a host batch; every byte through the 1-byte fold; short haystacks of every
    block count 0..5 and tail residue.  find_all of the class keys reports at each letter exactly the key of its class."""
    import torch
    keys, ids = class_keys()
    A = build(keys)
    cta_limit(A, limit)
    every = list(range(0x110000)) + [0x110000, 0x110001, 0x1FFFFF, 0x7FFFFFFF, 0xFFFFFFFF]
    flat, offs = wide_pair([every])
    want = [(0, e, k) for e, k in want_single(every, ids)]
    assert len(want) == len(_unicode_fold_map()[0]) + len(ids)
    assert triples(A.find_all_batch((flat, offs), case_insensitive=True)) == want
    d = torch.from_numpy(flat.reshape(1, -1).copy()).cuda()
    assert triples(A.find_all_batch(d, case_insensitive=True)) == want
    assert np.array_equal(d.cpu().numpy().reshape(-1), flat)                  # the caller's tensor is not changed
    latin = [list(range(256))]
    assert triples(A.find_all_batch([text(latin[0])], case_insensitive=True)) == \
        [(0, e, k) for e, k in want_single(latin[0], ids)]
    frm = _unicode_fold_map()[0]
    changed = frm[frm >= 256].tolist()
    for n in range(24):                                                       # 4-byte: n16 = 0..5, every tail
        hays = [changed[7 * n:7 * n + n], list(range(0xC0, 0xC0 + n))]
        got = triples(A.find_all_batch(wide_pair(hays), case_insensitive=True))
        assert got == [(h, e, k) for h, hay in enumerate(hays) for e, k in want_single(hay, ids)], n
    for n in range(96):                                                       # 1-byte: n16 = 0..5, every tail
        hays = [list(range(0xC0, 0x100))[:n] + [0x41] * max(0, n - 64)]
        got = triples(A.find_all_batch([text(h) for h in hays], case_insensitive=True))
        assert got == [(h, e, k) for h, hay in enumerate(hays) for e, k in want_single(hay, ids)], n


def device_batch(hays):
    """an equal-length batch as a CUDA tensor [n, stride] of 4-byte letters, or None"""
    import torch
    if not hays or len({len(h) for h in hays}) != 1 or not hays[0]:
        return None
    return torch.from_numpy(np.array(hays, dtype="<u4").view(np.uint8).reshape(len(hays), -1).copy()).cuda()


def check_methods(A, keys, hays, words=None, algo="auto"):
    """the four methods in every input form, and a CUDA tensor (left unchanged), against the restatement"""
    objs = [text(h) for h in hays]
    ww = False if words is None else text(sorted(words))
    is_word = None if words is None else words.__contains__
    kl = [len(k) for k in keys]
    full = eu.find_all(keys, hays)
    if is_word is not None:
        full = eu.whole_words(hays, full, kl, is_word)
    want = {"all": full, True: eu.leftmost(keys, hays, True, is_word), False: eu.leftmost(keys, hays, False, is_word)}
    reps = [[0x2A] * (i % 3) + [0x5F] for i in range(len(keys))]
    R = {first: A.replacer({text(k): text(r) for k, r in zip(keys, reps)}, leftmost_first=first) for first in (True, False)}
    batches = list(forms(objs, hays, 4, False))          # a latin-1 list takes the 1-byte route, the other forms 4 bytes
    d = device_batch(hays)
    if d is not None:
        batches.append(("device", d))
        before = d.clone()
    for form, b in batches:
        ctx = (form, keys, hays, words, algo)
        kw = dict(whole_words=ww, case_insensitive=True, algo=algo)
        assert triples(A.find_all_batch(b, **kw)) == want["all"], ctx
        assert sorted(triples(A.find_all_batch(b, sort=False, **kw))) == sorted(want["all"]), ctx
        assert triples(A.find_leftmost_first_batch(b, **kw)) == want[True], ctx
        assert triples(A.find_leftmost_longest_batch(b, **kw)) == want[False], ctx
        for first in (True, False):
            out = R[first].replace_batch(b, **kw)
            expect = eu.replace(keys, reps, hays, first, is_word)
            if form == "list":
                assert out == [text(x) for x in expect], ctx
            else:
                flat, offs = (x.cpu().numpy() if hasattr(x, "cpu") else x for x in out)
                assert [flat[offs[i]:offs[i + 1]].view("<u4").tolist() for i in range(len(hays))] == expect, ctx
    if d is not None:
        assert bool((d == before).all())


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["latin1", "wide", "mixed"])
@pytest.mark.parametrize("with_words", [False, True])
@pytest.mark.parametrize("algo", ["filter", "dfa"])
def test_gpu_every_route(case, with_words, algo):
    rng = np.random.default_rng(7 + len(case) + 2 * with_words + len(algo))
    alphabet = LATIN1 if case == "latin1" else TRAPS
    for _ in range(8):
        keys, hays = random_case(rng, alphabet)
        if case == "mixed":
            hays = [[c for c in h if c < 256] for h in hays] + [[0x10400, 0x41, 0x3C2]]
        if rng.integers(0, 2):
            hays = [h[:8] + [0x61] * max(0, 8 - len(h)) for h in hays]          # equal lengths: arrays and tensors
        words = set(int(x) for x in rng.choice(alphabet, size=4)) if with_words else None
        check_methods(build(keys), keys, hays, words, algo)


@pytest.mark.gpu
def test_gpu_pipelined_host_route_past_one_chunk():
    """a host batch of more than one 32 MiB chunk, latin-1 (1-byte letters) and wide, without case variants (the
    pipelined route): what the case-sensitive scan finds in the text folded beforehand"""
    rng = np.random.default_rng(23)
    frm, to = _unicode_fold_map()
    fold = dict(zip(frm.tolist(), to.tolist()))
    for alphabet, n in ((LATIN1, 40 << 20), (TRAPS, 9 << 20)):
        keys = sorted({text(rng.choice(alphabet, size=3).tolist()).translate(fold) for _ in range(12)})
        A = build([list(map(ord, k)) for k in keys])
        letters = rng.choice(np.array(alphabet, dtype=np.uint32), size=n)
        hays = np.array_split(letters, 3)
        if max(alphabet) < 256:                           # a list of latin-1 str: 1-byte letters
            batch = [h.astype(np.uint8).tobytes().decode("latin-1") for h in hays]
            folded = [eu.fold(h).astype(np.uint8).tobytes().decode("latin-1") for h in hays]
            assert sum(map(len, batch)) > 32 << 20
        else:
            offs = np.cumsum([0] + [4 * len(h) for h in hays]).astype(np.int64)
            batch = (np.concatenate(hays).astype("<u4").view(np.uint8), offs)
            folded = (eu.fold(np.concatenate(hays)).astype("<u4").view(np.uint8), offs)
            assert batch[0].size > 32 << 20
        got = A.find_all_batch(batch, case_insensitive=True)
        want = A.find_all_batch(folded)
        assert len(got) > 1000 and triples(got) == triples(want)


@pytest.mark.gpu
def test_gpu_ascii_text_as_the_ascii_fold():
    """ASCII keys and text: every route gives what ascii_case_insensitive gives"""
    rng = np.random.default_rng(29)
    al = [0x61, 0x41, 0x62, 0x42, 0x63, 0x20]
    for _ in range(10):
        keys, hays = random_case(rng, al)
        A = build(keys)
        hays_o = [text(h) for h in hays]
        d = device_batch([h[:8] + [0x61] * max(0, 8 - len(h)) for h in hays])
        for b in (hays_o, d):
            for m in ("find_all_batch", "find_leftmost_longest_batch", "find_leftmost_first_batch"):
                for ww in (False, True):
                    f = getattr(A, m)
                    assert triples(f(b, whole_words=ww, case_insensitive=True)) == triples(f(b, whole_words=ww, ascii_case_insensitive=True))
            R = A.replacer({text(k): "<%d>" % i for i, k in enumerate(keys)})
            u, a = R.replace_batch(b, case_insensitive=True), R.replace_batch(b, ascii_case_insensitive=True)
            if isinstance(b, list):
                assert u == a
            else:
                assert all(bool((x == y).all()) for x, y in zip(u, a))


@pytest.mark.gpu
@pytest.mark.parametrize("variants", [False, True])
def test_gpu_launch_counts(variants):
    """one fold launch before every scan; two more (count, scatter) for the expansion, on find_all with case variants"""
    import torch
    keys = ["σοφία", "straße", "müller"] + (["ΣΟΦΊΑ"] if variants else [])
    hays = ["ΣΟΦΊΑ and STRAẞE", "MÜLLER", "", "σοφία straße"]
    A = build([list(map(ord, k)) for k in keys])
    L = N.lib()
    d = torch.from_numpy(np.array([list(map(ord, h.ljust(16))) for h in hays], dtype="<u4").view(np.uint8).copy()).cuda()

    def count(call):
        call()                                                # every workspace grown
        before = L.acb_launch_count()
        call()
        return L.acb_launch_count() - before

    for b in (hays, d):
        plain = count(lambda: A.find_all_batch(b))
        assert count(lambda: A.find_all_batch(b, case_insensitive=True)) == plain + 1 + (2 if variants else 0)
        plain = count(lambda: A.find_leftmost_first_batch(b))
        assert count(lambda: A.find_leftmost_first_batch(b, case_insensitive=True)) == plain + 1
        plain = count(lambda: A.find_leftmost_longest_batch(b))
        assert count(lambda: A.find_leftmost_longest_batch(b, case_insensitive=True)) == plain + 1


@pytest.mark.gpu
def test_gpu_c_entry_refuses_bad_maps():
    A = build([[0x61, 0x62]])
    trie, lib = A._fold_host(False, _FOLD_UNICODE).trie, N.lib()
    narrow = A._fold_host(True, _FOLD_UNICODE).trie

    def upload(t, frm, to):
        tb = ctypes.c_void_p()
        frm, to = np.array(frm, dtype=np.uint32), np.array(to, dtype=np.uint32)
        rc = lib.acb_table_upload_folded_map(t, 0, None, None, 0, N.ptr(frm), N.ptr(to), len(frm), ctypes.byref(tb))
        if rc == N.ACB_OK:
            lib.acb_table_free(tb)
        return rc
    assert upload(trie, [0x41, 0x42], [0x21, 0x21]) == N.ACB_OK
    assert upload(trie, [0x42, 0x41], [0x21, 0x21]) == N.ACB_EINVAL                  # not ascending
    assert upload(trie, [0x41, 0x41], [0x21, 0x21]) == N.ACB_EINVAL                  # not strictly
    assert upload(trie, [0x41], [0x61]) == N.ACB_EINVAL                              # to above from
    assert upload(trie, [0x41, 0x61], [0x21, 0x41]) == N.ACB_EINVAL                  # a to that is itself mapped
    assert upload(trie, [0x110000], [0x41]) == N.ACB_EINVAL                          # not a code point
    assert upload(narrow, [0x41, 0x212A], [0x21, 0x4B]) == N.ACB_OK                  # from >= 256 may go below 256
    assert upload(narrow, [0xC9], [0x41]) == N.ACB_OK
    frm = np.array([0x100 * (b + 1) for b in range(43)], dtype=np.uint32)            # 43 changing blocks: too many
    assert upload(trie, frm, frm - 1) == N.ACB_EINVAL and upload(trie, frm[:42], frm[:42] - 1) == N.ACB_OK
    fm, tm = _unicode_fold_map()
    assert upload(narrow, fm, tm) == N.ACB_OK and upload(trie, fm, tm) == N.ACB_OK


@pytest.mark.gpu
def test_gpu_past_2_gib():
    """A CUDA tensor of 4-byte letters past 2^31 bytes (520 rows of 4 MiB + 64): keys in every case at row edges, around
    byte 2^31 and inside rows, with case variants (the expansion runs); find_all checked by construction."""
    import torch
    stride = (1 << 20) + 16                                                      # letters per row
    n_rows = 520
    assert n_rows * stride * 4 > (1 << 31) + (1 << 24)
    keys = ["σοφία", "ΣΟΦΊΑ", "straße"]
    plants = {0: "ΣΟΦΊΑ", 1: "STRAẞE", 2: "σοφία", 3: "Straße"}
    A = build([list(map(ord, k)) for k in keys])
    t = torch.full((n_rows, stride), 0x78, dtype=torch.int32, device="cuda")
    G = (1 << 31) // 4                                                            # letter index of byte 2^31
    want = []
    spots = []
    for r in range(n_rows):
        spots += [(r, 0), (r, stride - 6), (r, 1000 + r)]
    r31, c31 = divmod(G, stride)
    spots += [(r31, c31 - 3), (r31, c31 + 9)] if c31 >= 3 and c31 + 15 < stride else []
    for i, (r, c) in enumerate(sorted(set(spots))):
        w = plants[i % 4]
        t[r, c:c + len(w)] = torch.tensor([ord(x) for x in w], dtype=torch.int32)
        ids = [0, 1] if i % 2 == 0 else [2]                                       # σοφία and ΣΟΦΊΑ, or straße
        want += [(r, c + len(w) - 1, k) for k in ids]
    got = A.find_all_batch(t.view(torch.uint8), case_insensitive=True)
    assert triples(got) == sorted(want)
