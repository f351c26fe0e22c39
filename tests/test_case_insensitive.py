"""ascii_case_insensitive=True of find_all_batch, find_leftmost_longest_batch, find_leftmost_first_batch and
Replacer.replace_batch: keys and text compared with the 26 ASCII capitals made small, the text folded on the GPU, the
word test and the rewrite on the text as given.

The CPU half checks the restatement (tests/emul_fold.py) against Python's `re` with IGNORECASE | ASCII, the key groups
the Automaton builds, the alias expansion and the refusals; the gpu-marked half runs the real routes against the
restatement, the C oracle and the case-sensitive routes over folded text."""
import ctypes
import re

import numpy as np
import pytest

import emul_fold as ef
import oracle
import pyahocorasick_b200 as pkg
from batch_cases import forms, obj, triples
from pyahocorasick_b200 import _native as N

FLAGS = re.IGNORECASE | re.ASCII
# letters beside the ASCII ones that must not fold: the neighbours of A-Z and a-z, latin-1 and wider capitals/smalls
TRAPS = {"bytes": [0x40, 0x60, 0x5B, 0x7B, 0xC1, 0xE1],
         "latin1": [0x40, 0x60, 0x5B, 0x7B, 0xC9, 0xE9],
         "wide": [0x141, 0x161, 0xC9, 0xE9, 0x1F641, 0x1F661],
         "mixed": [0x40, 0xC9, 0xE9, 0x1F641]}
FLAVOUR = {"bytes": "bytes", "latin1": "unicode", "wide": "unicode", "mixed": "unicode"}


def alphabet(case):
    return [0x61, 0x41, 0x62, 0x42] + TRAPS[case]


def random_case(case, rng, n_keys=None, n_hays=None):
    al = alphabet(case)
    keys = []
    for _ in range(n_keys or int(rng.integers(1, 9))):
        k = [int(x) for x in rng.choice(al, size=int(rng.integers(1, 5)))]
        if k not in keys:
            keys.append(k)
        if rng.integers(0, 3) == 0:                              # a case variant of it
            v = [x ^ 0x20 if 0x41 <= (x | 0x20) - 0x20 <= 0x5A else x for x in k]
            if v not in keys:
                keys.append(v)
    hays = [[int(x) for x in rng.choice(al, size=int(rng.integers(0, 40)))] for _ in range(n_hays or int(rng.integers(1, 6)))]
    if case == "mixed" and all(max(h, default=0) < 256 for h in hays):
        hays.append([0x1F600, 0x61, 0x41])
    return keys, hays


def text(fl, letters):
    return obj(fl, False, letters)


def build(fl, keys):
    """the Automaton (STORE_INTS, value = key id) over keys given as letters, None for an id left unused"""
    mod = pkg.flavour(fl)
    A = mod.Automaton(mod.STORE_INTS)
    for i, k in enumerate(keys):
        A.add_word(text(fl, k if k is not None else [0x7E] * (i + 40)), i)
    for i, k in enumerate(keys):
        if k is None:
            A.remove_word(text(fl, [0x7E] * (i + 40)))
    A.make_automaton()
    return A


# ------------------------------------------------------------------ `re` (CPU)
def re_escape(fl, letters):
    return re.escape(text(fl, letters))


def re_find_all(fl, keys, hays):
    out = []
    for h, hay in enumerate(hays):
        t = text(fl, hay)
        for kid, k in enumerate(keys):
            for m in re.finditer((b"(?=" if fl == "bytes" else "(?=") + re_escape(fl, k) + (b")" if fl == "bytes" else ")"), t, FLAGS):
                out.append((h, m.start() + len(k) - 1, -len(k), kid))
    return [(h, e, k) for h, e, _, k in sorted(out)]


def re_pattern(fl, keys, order, words=None):
    """the alternation of the keys in `order`, one group each; with a word set, between look-arounds on its letters"""
    sep, grp = (b"|", lambda s: b"(" + s + b")") if fl == "bytes" else ("|", lambda s: "(" + s + ")")
    alt = sep.join(grp(re_escape(fl, keys[i])) for i in order)
    if words is not None:
        cls = text(fl, sorted(words))
        if cls:                                               # the word letters exactly as given: case-sensitive classes
            cls = re.escape(cls)
            alt = (b"(?<!(?-i:[%s]))(?:%s)(?!(?-i:[%s]))" % (cls, alt, cls)) if fl == "bytes" else \
                f"(?<!(?-i:[{cls}]))(?:{alt})(?!(?-i:[{cls}]))"
    return re.compile(alt, FLAGS)


def orders(keys):
    first = list(range(len(keys)))
    return {True: first, False: sorted(first, key=lambda i: (-len(keys[i]), i))}


def re_leftmost(fl, keys, hays, first, words=None):
    order = orders(keys)[first]
    pat = re_pattern(fl, keys, order, words)
    return [(h, m.end() - 1, order[m.lastindex - 1]) for h, hay in enumerate(hays) for m in pat.finditer(text(fl, hay))]


def re_replace(fl, keys, reps, hays, first, words=None):
    order = orders(keys)[first]
    pat = re_pattern(fl, keys, order, words)
    return [pat.sub(lambda m: text(fl, reps[order[m.lastindex - 1]]), text(fl, hay)) for hay in hays]


def test_swar_fold_is_the_definition():
    lanes = np.arange(256, dtype=np.uint32)
    for shift in (0, 8, 16, 24):
        w = ef.fold_swar((lanes << np.uint32(shift)) | np.uint32(0x5A41C15B & ~(0xFF << shift)))
        assert np.array_equal((w >> np.uint32(shift)) & np.uint32(0xFF), ef.fold(lanes))
    words = np.random.default_rng(0).integers(0, 2 ** 32, size=1 << 16, dtype=np.uint32)
    want = ef.fold(words.view(np.uint8)).astype(np.uint8).view(np.uint32)
    assert np.array_equal(ef.fold_swar(words), want)


@pytest.mark.parametrize("case", ["bytes", "latin1", "wide"])
def test_definitions_agree_with_re(case):
    fl = FLAVOUR[case]
    rng = np.random.default_rng(len(case))
    for _ in range(150):
        keys, hays = random_case(case, rng)
        assert ef.find_all(keys, hays) == re_find_all(fl, keys, hays), (keys, hays)
        reps = [[0x5F] * int(rng.integers(0, 3)) + k[:1] for k in keys]
        words = set(int(x) for x in rng.choice(alphabet(case), size=3))
        for first in (True, False):
            assert ef.leftmost(keys, hays, first) == re_leftmost(fl, keys, hays, first), (keys, hays, first)
            assert [text(fl, x) for x in ef.replace(keys, reps, hays, first)] == re_replace(fl, keys, reps, hays, first)
            is_word = words.__contains__
            assert ef.leftmost(keys, hays, first, is_word) == re_leftmost(fl, keys, hays, first, words), (keys, hays, words)
            assert [text(fl, x) for x in ef.replace(keys, reps, hays, first, is_word)] == \
                re_replace(fl, keys, reps, hays, first, words)


def test_examples():
    keys = [list(b"abc"), list(b"ABC")]
    assert ef.find_all(keys, [list(b"xAbCx")]) == [(0, 3, 0), (0, 3, 1)]
    assert ef.leftmost(keys, [list(b"xAbCx")], True) == [(0, 3, 0)]
    assert ef.leftmost([list(b"x")], [list(b"Ax"), list(b"ax")], True, set(b"abc").__contains__) == [(0, 1, 0)]
    assert ef.replace([list(b"secret")], [list(b"***")], [list(b"A Secret, SECRET.")], False) == [list(b"A ***, ***.")]


def keys_in(A, core, fl):
    """the (folded key, id) pairs of a folded host trie, found through acb_trie_find"""
    lib = A._lib
    got = {}
    for kid, key in enumerate(A._key_objs):
        if key is None:
            continue
        raw, _ = A._raw_key(pkg.automaton._ascii_fold(key))
        k, pre = ctypes.c_int32(-1), ctypes.c_int32(0)
        N.check(lib.acb_trie_find(core.trie, raw, len(raw), ctypes.byref(k), ctypes.byref(pre)))
        got[raw] = k.value
    assert lib.acb_trie_count(core.trie) == len(got)
    return got


@pytest.mark.parametrize("fl", ["bytes", "unicode"])
def test_folded_trie_holds_representatives(fl):
    mod = pkg.flavour(fl)
    A = mod.Automaton(mod.STORE_INTS)
    t = (lambda s: s.encode("latin-1")) if fl == "bytes" else (lambda s: s)
    words = ["abc", "ABC", "Abc", "x", "X", "É", "é"] + ([] if fl == "bytes" else ["Łx", "šx", "aBc\U0001F641"])
    for i, w in enumerate(words):
        A.add_word(t(w), i)
    A.make_automaton()
    core = A._fold_host(False)
    got = keys_in(A, core, fl)
    want_rep, want_alias = ef.groups([list(t(w)) if fl == "bytes" else list(map(ord, w)) for w in words])
    assert sorted(set(got.values())) == sorted(set(want_rep.values()))
    ptr, ids = ef.alias_csr([list(t(w)) if fl == "bytes" else list(map(ord, w)) for w in words])
    assert core.alias_ptr.tolist() == ptr.tolist() and core.alias_ids.tolist() == ids.tolist()
    assert want_alias == {0: [1, 2], 3: [4]}                # É and é, Ł and š stay apart
    if fl == "unicode":
        assert A._fold_host(True).alias_ids.tolist() == [1, 2, 4]     # the latin-1 keys
    # the representative moves when the lowest id goes, and a key added again comes last
    A.remove_word(t("abc"))
    A.make_automaton()
    assert A._fold_host(False).alias_ids.tolist()[:1] == [2] and keys_in(A, A._fold_host(False), fl)[t("abc") if fl == "bytes" else "abc".encode("utf-32-le")] == 1
    A.add_word(t("abc"), 99)
    A.make_automaton()
    core = A._fold_host(False)
    rep = keys_in(A, core, fl)[t("abc") if fl == "bytes" else "abc".encode("utf-32-le")]
    assert rep == 1 and core.alias_ids[core.alias_ptr[1]:core.alias_ptr[2]].tolist() == [2, len(words)]


def test_expansion_restated():
    rng = np.random.default_rng(3)
    for _ in range(50):
        keys, _ = random_case("bytes", rng, n_keys=12)
        ptr, ids = ef.alias_csr(keys)
        rep, aliases = ef.groups(keys)
        reps = sorted(set(rep.values()))
        rec = np.array([(int(rng.integers(0, 4)), int(rng.integers(0, 50)), int(rng.choice(reps))) for _ in range(30)])
        want = [(h, e, k) for h, e, r in rec.tolist() for k in [r] + aliases.get(r, [])]
        got, total = ef.expand(rec, ptr, ids, 10 ** 6)
        assert total == len(want) and [tuple(x) for x in got.tolist()] == want
        assert ef.expand(rec, ptr, ids, 5)[1] == total


def test_refusals():
    A = build("bytes", [list(b"ab")])
    for call in (lambda: A.find_all_batch([b"ab"], ignore_white_space=True, ascii_case_insensitive=True),
                 lambda: A.find_all_batch([b"ab"], algo="long", ascii_case_insensitive=True),
                 lambda: A.find_long_batch([b"ab"], ascii_case_insensitive=True)):
        with pytest.raises(ValueError):
            call()
    mod = pkg.flavour("unicode")
    S = mod.Automaton(mod.STORE_INTS, mod.KEY_SEQUENCE)
    S.add_word((1, 2), 0)
    S.make_automaton()
    for call in (lambda: S.find_all_batch([(1, 2)], ascii_case_insensitive=True),
                 lambda: S.find_leftmost_longest_batch([(1, 2)], ascii_case_insensitive=True),
                 lambda: S.find_leftmost_first_batch([(1, 2)], ascii_case_insensitive=True)):
        with pytest.raises(ValueError, match="KEY_SEQUENCE"):
            call()
    import inspect
    for m in (A.stream_batch, pkg.automaton.Replacer.stream_batch, A.iter):
        assert "ascii_case_insensitive" not in inspect.signature(m).parameters


# ------------------------------------------------------------------ the GPU
def device_batch(fl, hays):
    """an equal-length batch as a CUDA tensor [n, stride] at the flavour's full letter width, or None"""
    import torch
    if not hays or len({len(h) for h in hays}) != 1 or not hays[0]:
        return None
    a = np.array(hays, dtype=np.uint8 if fl == "bytes" else "<u4")
    return torch.from_numpy(a.view(np.uint8).reshape(len(hays), -1).copy()).cuda()


def check_methods(A, case, keys, hays, words=None):
    """the four methods in every input form, and a CUDA tensor, against the restatement"""
    fl = FLAVOUR[case]
    objs = [text(fl, h) for h in hays]
    ww = False if words is None else text(fl, sorted(words))
    is_word = None if words is None else words.__contains__
    full = ef.find_all(keys, hays)
    if is_word is not None:
        full = ef.whole_words(hays, full, ef.key_lengths(keys), is_word)
    want = {"all": full, True: ef.leftmost(keys, hays, True, is_word), False: ef.leftmost(keys, hays, False, is_word)}
    reps = [None if k is None else [0x2A] * (i % 3) + [0x5F] for i, k in enumerate(keys)]
    R = {first: A.replacer({text(fl, k): text(fl, r) for k, r in zip(keys, reps) if k is not None}, leftmost_first=first)
         for first in (True, False)}
    batches = list(forms(objs, hays, A._L, case in ("latin1", "mixed")))
    d = device_batch(fl, hays)
    if d is not None:
        batches.append(("device", d))
    for form, b in batches:
        ctx = (case, form, keys, hays, words)
        assert triples(A.find_all_batch(b, whole_words=ww, ascii_case_insensitive=True)) == want["all"], ctx
        assert triples(A.find_leftmost_first_batch(b, whole_words=ww, ascii_case_insensitive=True)) == want[True], ctx
        assert triples(A.find_leftmost_longest_batch(b, whole_words=ww, ascii_case_insensitive=True)) == want[False], ctx
        unsorted = A.find_all_batch(b, whole_words=ww, ascii_case_insensitive=True, sort=False)
        assert sorted(triples(unsorted)) == sorted(want["all"]), ctx
        for first in (True, False):
            out = R[first].replace_batch(b, whole_words=ww, ascii_case_insensitive=True)
            expect = ef.replace(keys, reps, hays, first, is_word)
            if form == "list":
                assert out == [text(fl, x) for x in expect], ctx
            else:
                flat, offs = (x.cpu().numpy() if hasattr(x, "cpu") else x for x in out)
                L = 1 if (fl == "bytes" or (form != "device" and A._L == 1)) else 4
                dt = np.uint8 if L == 1 else "<u4"
                got = [flat[offs[i]:offs[i + 1]].view(dt).tolist() for i in range(len(hays))]
                assert got == expect, ctx


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["bytes", "latin1", "wide", "mixed"])
@pytest.mark.parametrize("with_words", [False, True])
def test_gpu_every_form(case, with_words):
    rng = np.random.default_rng(11 + len(case) + with_words)
    fl = FLAVOUR[case]
    for _ in range(12):
        keys, hays = random_case(case, rng)
        if rng.integers(0, 2):
            hays = [h[:8] + [0x61] * max(0, 8 - len(h)) for h in hays]          # equal lengths: arrays and tensors
        A = build(fl, keys)
        words = set(int(x) for x in rng.choice(alphabet(case), size=3)) if with_words else None
        check_methods(A, case, keys, hays, words)


@pytest.mark.gpu
@pytest.mark.parametrize("placement", ["pair", "single", "dfa", "cta1"])
def test_gpu_filter_placements(monkeypatch, placement):
    """the same answers whichever kernel scans: the pair and single filters forced, the DFA, a one-CTA grid"""
    if placement in ("pair", "single"):
        monkeypatch.setenv("ACB_FILTER", "4,1,0,1" if placement == "pair" else "4,1,0,0")
    rng = np.random.default_rng(5)
    al = [0x61, 0x41, 0x62, 0x42, 0x40, 0x60, 0xC1, 0xE1]
    keys = []
    while len(keys) < 40:
        k = [int(x) for x in rng.choice(al, size=int(rng.integers(4, 9)))]
        keys += [k, [x ^ 0x20 if (x | 0x20) in (0x61, 0x62) else x for x in k]] if k not in keys else []
    hays = [[int(x) for x in rng.choice(al[:4], size=3000)] for _ in range(3)] + [[int(x) for x in rng.choice(al, size=500)]]
    A = build("bytes", keys)
    algo = "dfa" if placement == "dfa" else "auto"
    tb = A._table_for(0, False, True)
    if placement == "cta1":
        N.check(A._lib.acb_table_set_cta_limit(tb, 1))
    fv = N.FlatView()
    N.check(A._lib.acb_trie_flat_view(A._fold_host(False).trie, ctypes.byref(fv)))
    if placement in ("pair", "single"):
        assert bool(fv.filter_flags & 2) == (placement == "pair") and fv.gram_bytes == 4
    objs = [text("bytes", h) for h in hays]
    assert triples(A.find_all_batch(objs, algo=algo, ascii_case_insensitive=True)) == ef.find_all(keys, hays)
    assert triples(A.find_leftmost_first_batch(objs, algo=algo, ascii_case_insensitive=True)) == ef.leftmost(keys, hays, True)
    assert triples(A.find_leftmost_longest_batch(objs, algo=algo, ascii_case_insensitive=True)) == ef.leftmost(keys, hays, False)
    short = [h[:500] for h in hays]
    d = device_batch("bytes", short)
    assert triples(A.find_all_batch(d, algo=algo, ascii_case_insensitive=True)) == ef.find_all(keys, short)
    assert triples(A.find_leftmost_first_batch(d, algo=algo, ascii_case_insensitive=True)) == ef.leftmost(keys, short, True)


@pytest.mark.gpu
def test_gpu_trap_letters_do_not_fold():
    for case in ("bytes", "latin1", "wide"):
        fl = FLAVOUR[case]
        keys = [[t] for t in TRAPS[case]] + [[0x61], [0x5A]]
        hays = [TRAPS[case] + [x ^ 0x20 for x in TRAPS[case] if x < 0x100] + [0x41, 0x7A], [0x1F641, 0x141, 0xC1, 0x61] if case == "wide" else [0xC1, 0x61]]
        A = build(fl, keys)
        check_methods(A, case, keys, hays)


@pytest.mark.gpu
def test_gpu_groups_up_to_64_variants_and_the_capacity_retry():
    """every case variant of aaaaaa added in shuffled order: the lowest id wins, find_all gives the group in ascending id;
    the text holds enough matches that both the host and the device route overflow their first capacity once"""
    import itertools
    import torch
    rng = np.random.default_rng(64)
    variants = [list(v) for v in itertools.product(*[(0x61, 0x41)] * 6)]
    order = rng.permutation(len(variants))
    for size in (1, 2, 7, 64):
        keys = [variants[i] for i in order[:size]] + [list(b"bab")]
        hays = [[int(x) for x in rng.choice([0x61, 0x41, 0x62], size=300)] for _ in range(4)] + [[0x41] * 200]
        A = build("bytes", keys)
        A._match_cap = 0
        want = ef.find_all(keys, hays)
        if size == 64:
            assert len(want) > 4096                          # more than the first capacity
        assert triples(A.find_all_batch([text("bytes", h) for h in hays], ascii_case_insensitive=True)) == want
        assert A.find_leftmost_first_batch([text("bytes", h) for h in hays], ascii_case_insensitive=True).key_id.tolist() == \
            [k for _, _, k in ef.leftmost(keys, hays, True)]
        A._match_cap = 0
        d = torch.from_numpy(np.array([h[:200] for h in hays], dtype=np.uint8)).cuda()
        assert triples(A.find_all_batch(d, ascii_case_insensitive=True)) == ef.find_all(keys, [h[:200] for h in hays])


@pytest.mark.gpu
def test_gpu_words_are_tested_in_the_text_as_given():
    A = build("bytes", [list(b"x")])
    for b in ([b"Ax", b"ax", b"xA", b"AxB"], device_batch("bytes", [list(b"Ax"), list(b"ax")])):
        got = triples(A.find_all_batch(b, whole_words=b"abc", ascii_case_insensitive=True))
        assert got == [(0, 1, 0)] + ([(2, 0, 0), (3, 1, 0)] if isinstance(b, list) else [])


@pytest.mark.gpu
def test_gpu_replacement_keeps_the_case_of_the_text():
    A = pkg.flavour("bytes").Automaton()
    for i, k in enumerate([b"secret", b"Secret", b"KEY"]):
        A.add_word(k, i)
    A.make_automaton()
    R = A.replacer({b"secret": b"[s]", b"Secret": b"[S]", b"KEY": b"[k]"})
    got = R.replace_batch([b"My Secret Key, SECRET and secret; keyS.", b"NoNe"], ascii_case_insensitive=True)
    assert got == [b"My [s] [k], [s] and [s]; [k]S.", b"NoNe"]
    assert R.replace_batch([b"My Secret Key"]) == [b"My [S] Key"]
    U = pkg.flavour("unicode").Automaton()
    U.add_word("été", 0)
    U.make_automaton()
    assert U.replacer({"été": "x"}).replace_batch(["ÉTÉ éTé"], ascii_case_insensitive=True) == \
        ["ÉTÉ x"]


@pytest.mark.gpu
def test_gpu_case_sensitive_calls_between_and_add_word_after():
    A = build("bytes", [list(b"he"), list(b"HE"), list(b"she")])
    hays = [b"She said HE, he, hE", b"SHE"]
    plain = triples(A.find_all_batch(hays))
    folded = triples(A.find_all_batch(hays, ascii_case_insensitive=True))
    longest = triples(A.find_leftmost_longest_batch(hays))
    for _ in range(2):
        assert triples(A.find_all_batch(hays)) == plain
        assert triples(A.find_all_batch(hays, ascii_case_insensitive=True)) == folded
        assert triples(A.find_leftmost_longest_batch(hays)) == longest
    assert folded == ef.find_all([list(b"he"), list(b"HE"), list(b"she")], [list(h) for h in hays])
    assert plain != folded
    A.add_word(b"SAID", 3)
    A.make_automaton()
    keys = [list(b"he"), list(b"HE"), list(b"she"), list(b"SAID")]
    assert triples(A.find_all_batch(hays, ascii_case_insensitive=True)) == ef.find_all(keys, [list(h) for h in hays])


# launches: the fold is one launch before every scan; the alias expansion two (count, scatter) after it, only on a key set
# with case variants and only on the find_all routes
FOLD, EXPAND = 1, 2
SORT = 1                                                      # the sort key of a one-pass device sort


@pytest.mark.gpu
@pytest.mark.parametrize("variants", [False, True])
def test_gpu_launch_counts(variants):
    import torch
    keys = [b"he", b"she", b"his", b"hers"] + ([b"HE"] if variants else [])
    hays = [b"ushers and SHE sells his shells", b"his hers", b"", b"hehe she said"]
    A = pkg.flavour("bytes").Automaton()
    for i, k in enumerate(keys):
        A.add_word(k, i)
    A.make_automaton()
    L = N.lib()
    d = torch.from_numpy(np.frombuffer(b"".join(h.ljust(32) for h in hays), dtype=np.uint8).reshape(4, 32).copy()).cuda()

    def count(call):
        call()                                                # every workspace grown
        before = L.acb_launch_count()
        call()
        return L.acb_launch_count() - before

    for b in (hays, d):
        plain = count(lambda: A.find_all_batch(b))
        assert count(lambda: A.find_all_batch(b, ascii_case_insensitive=True)) == plain + FOLD + (EXPAND if variants else 0)
        plain = count(lambda: A.find_leftmost_first_batch(b))
        assert count(lambda: A.find_leftmost_first_batch(b, ascii_case_insensitive=True)) == plain + FOLD
        assert count(lambda: A.find_leftmost_first_batch(b)) == plain       # the case-sensitive route as before


@pytest.mark.gpu
def test_gpu_c_entries_refuse_and_expand():
    import torch
    A = build("bytes", [list(b"ab"), list(b"AB"), list(b"Ab")])
    L = N.lib()
    plain = A._ensure_table(0)                                 # first: a first upload of the plain table drops the others
    tb = A._table_for(0, False, True)
    found = ctypes.c_int64()
    flat = np.frombuffer(b"xaBx", dtype=np.uint8).copy()
    assert L.acb_scan_host(tb, N.ptr(flat), 4, None, 1, 4, None, 16, ctypes.byref(found), N.ALGO_LONG, 1) == N.ACB_EINVAL
    ss = ctypes.c_void_p()
    assert L.acb_streams_new(tb, 1, 0, ctypes.byref(ss)) == N.ACB_EINVAL
    key_id, prefix = np.empty(1, np.int32), np.empty(1, np.int32)
    assert L.acb_lookup_host(tb, N.ptr(flat), 4, None, 1, 4, N.ptr(key_id), N.ptr(prefix)) == N.ACB_EINVAL
    skip = np.array([32], dtype=np.uint32)
    assert L.acb_scan_host_skip(tb, N.ptr(flat), 4, None, 1, 4, None, 16, ctypes.byref(found), 0, 1, N.ptr(skip), 1) == N.ACB_EINVAL
    cnt = torch.zeros(1, dtype=torch.int64, device="cuda")
    assert L.acb_expand_aliases_device(plain, None, 0, None, 0, cnt.data_ptr(), None) == N.ACB_EINVAL
    tb2 = ctypes.c_void_p()
    bad = np.array([0, 2], dtype=np.int32)
    ids = np.array([2, 1], dtype=np.int32)                     # not ascending
    assert L.acb_table_upload_folded(A._fold_host(False).trie, 0, N.ptr(bad), N.ptr(ids), 2, ctypes.byref(tb2)) == N.ACB_EINVAL
    rec = torch.tensor([[0, 2, 0], [1, 5, 0], [1, 6, 9]], dtype=torch.int32, device="cuda")
    for cap in (0, 2, 7):
        out = torch.full((max(cap, 1), 3), -7, dtype=torch.int32, device="cuda")
        cnt = torch.full((1,), 99, dtype=torch.int64, device="cuda")
        N.check(L.acb_expand_aliases_device(tb, rec.data_ptr(), 3, out.data_ptr(), cap, cnt.data_ptr(),
                                            torch.cuda.current_stream().cuda_stream))
        want, total = ef.expand(rec.cpu().numpy(), *ef.alias_csr([list(b"ab"), list(b"AB"), list(b"Ab")]), cap)
        assert int(cnt.item()) == total == 7
        assert out.cpu().numpy()[:min(cap, 7)].tolist() == want.tolist()


# ------------------------------------------------------------------ the workloads at full size
def _folded_reference(keys, hays2d):
    """the answers over folded text with a case-sensitive automaton of the folded group representatives"""
    rep, aliases = ef.groups([list(k) for k in keys])
    F = pkg.flavour("bytes").Automaton(pkg.flavour("bytes").STORE_INTS)
    for kid, k in enumerate(keys):
        if rep[kid] == kid:
            F.add_word(bytes(ef.fold(list(k)).astype(np.uint8)), kid)
    F.make_automaton()
    folded = ef.fold(hays2d).astype(np.uint8)
    out = {}
    m = F.find_all_batch(folded)
    full = np.stack([m.hay_id, m.end_index, np.array(m.values(), dtype=np.int64)], axis=1).astype(np.int64)
    ptr, aid = ef.alias_csr([list(k) for k in keys])
    out["all"] = full
    if len(aid):
        cnt = np.ones(len(full), dtype=np.int64)
        inside = full[:, 2] < len(ptr) - 1
        cnt[inside] += ptr[full[inside, 2] + 1] - ptr[full[inside, 2]]
        rows = np.repeat(full, cnt, axis=0)
        first = np.repeat(np.cumsum(cnt) - cnt, cnt)
        j = np.arange(len(rows)) - first - 1
        alias = j >= 0
        rows[alias, 2] = aid[ptr[rows[alias, 2]] + j[alias]]
        out["all"] = rows
    for first in (True, False):
        mm = F.find_leftmost_first_batch(folded) if first else F.find_leftmost_longest_batch(folded)
        out[first] = np.stack([mm.hay_id, mm.end_index, np.array(mm.values(), dtype=np.int64)], axis=1).astype(np.int64)
    return out, folded


@pytest.mark.gpu
@pytest.mark.parametrize("name,swapped", [("C2", False), ("C2", True), ("C4", False)])
def test_gpu_workloads_at_full_size(name, swapped):
    """case-flipped text; C2's keys, or C2's keys and every key's swapcase() (groups of two)"""
    import torch
    from pyahocorasick_b200 import synth
    from batch_cases import rows
    w = synth.make(name)
    keys = list(w.keys)
    if swapped:
        have = set(keys)
        keys += [k.swapcase() for k in w.keys if k.swapcase() not in have]
    rng = np.random.default_rng(17)
    hays = w.haystacks.copy()
    flip = rng.integers(0, 2, size=hays.shape).astype(bool) & (((hays | 0x20) >= 0x61) & ((hays | 0x20) <= 0x7A))
    hays[flip] ^= 0x20
    A = pkg.flavour("bytes").Automaton(pkg.flavour("bytes").STORE_INTS)
    for i, k in enumerate(keys):
        A.add_word(k, i)
    A.make_automaton()
    want, folded = _folded_reference(keys, hays)
    d = torch.from_numpy(hays).cuda()
    for b in (hays, d):
        assert np.array_equal(rows(A.find_all_batch(b, ascii_case_insensitive=True)), want["all"])
        assert np.array_equal(rows(A.find_leftmost_first_batch(b, ascii_case_insensitive=True)), want[True])
        assert np.array_equal(rows(A.find_leftmost_longest_batch(b, ascii_case_insensitive=True)), want[False])
    # a few thousand rows against the C oracle, over the folded text and the folded representatives
    rep, _ = ef.groups([list(k) for k in keys])
    O = oracle.OracleAutomaton()
    for kid, k in enumerate(keys):
        if rep[kid] == kid:
            O.add_word(bytes(ef.fold(list(k)).astype(np.uint8)), kid)
    O.make_automaton()
    n = 3000 if name == "C2" else 2                          # C2: 3000 x 256 B; C4: two 16 MiB haystacks
    sub = folded[:n]
    off = np.arange(n + 1, dtype=np.int64) * sub.shape[1]
    ref = sorted(map(tuple, O.scan_batch_bytes(sub.reshape(-1), off).tolist()))
    got = rows(A.find_all_batch(hays[:n], ascii_case_insensitive=True))
    got = sorted((h, e, k) for h, e, k in got.tolist() if rep[k] == k)
    assert got == ref
