"""ascii_case_insensitive_stream_batch of Automaton and Replacer: find_all, leftmost-longest, leftmost-first and replacing
streams (with and without whole words) that compare keys and text with the 26 ASCII capitals made small.

Whatever the chunking, a stream's feeds (plus its finish) must give exactly what the whole-batch method gives for its
whole text with ascii_case_insensitive=True: the definitions of tests/emul_fold.py (checked against `re` in
test_case_insensitive.py) on the CPU and in small GPU cases, the whole-batch methods themselves at scale.  The CPU tests
run the Python layer on the restatement of the folded feeds (tests/emul_stream_fold.py); the gpu-marked tests run the
real kernels."""
import ctypes

import numpy as np
import pytest

import emul_fold as ef
import emul_leftmost_first
import emul_stream_fold
import emul_stream_leftmost
import emul_streams
import pyahocorasick_b200 as pkg
from batch_cases import rows
from pyahocorasick_b200 import _native as N

# letters beside the ASCII ones that must not fold: the neighbours of A-Z and a-z, latin-1 and wider letters
TRAPS = {"bytes": [0x40, 0x5B, 0x60, 0x7B, 0xC1, 0xE1],
         "latin1": [0x40, 0x5B, 0x60, 0x7B, 0xC9, 0xE9],
         "wide": [0x141, 0x161, 0xC9, 0xE9, 0x1F641, 0x1F661],
         "mixed": [0x40, 0xC9, 0xE9, 0x1F641]}
FLAVOUR = {"bytes": "bytes", "latin1": "unicode", "wide": "unicode", "mixed": "unicode"}
# form -> (batch kind, leftmost-first, whole words)
FORMS = {"all": ("all", False, False), "all_words": ("all", False, True), "longest": ("leftmost", False, False),
         "first": ("leftmost", True, False), "longest_words": ("leftmost", False, True), "first_words": ("leftmost", True, True),
         "replace_longest": ("replace", False, False), "replace_first": ("replace", True, False),
         "replace_longest_words": ("replace", False, True)}
WORDS = [0x61, 0x41, 0x62]                                   # the word set of the whole-word forms: a, A and b as given


def text(fl, letters):
    return bytes(letters) if fl == "bytes" else "".join(map(chr, letters))


def build(fl, keys):
    """the Automaton (STORE_INTS, value = key id) over keys given as letters"""
    mod = pkg.flavour(fl)
    A = mod.Automaton(mod.STORE_INTS)
    for i, k in enumerate(keys):
        A.add_word(text(fl, k), i)
    A.make_automaton()
    return A


def variant(k):
    return [x ^ 0x20 if 0x41 <= (x & ~0x20) <= 0x5A else x for x in k]


def random_keys(case, rng, n=None):
    al = [0x61, 0x41, 0x62, 0x42] + TRAPS[case]
    keys = []
    for _ in range(n or int(rng.integers(1, 7))):
        k = [int(x) for x in rng.choice(al, size=int(rng.integers(1, 5)))]
        for v in ([k, variant(k)] if rng.integers(0, 2) else [k]):
            if v not in keys:
                keys.append(v)
    return keys


def random_text(case, keys, rng, n):
    al = [0x61, 0x41, 0x62, 0x42] + TRAPS[case]
    body = []
    while len(body) < n:
        body += variant(keys[int(rng.integers(0, len(keys)))]) if rng.integers(0, 2) else \
            [int(x) for x in rng.choice(al, size=int(rng.integers(1, 4)))]
    return body[:n]


def definition(form, keys, reps, seg):
    """what a stream of this form gives for its whole text `seg`: [(end, key id)] or the output letters"""
    kind, first, words = FORMS[form]
    is_word = set(WORDS).__contains__ if words else None
    if kind == "replace":
        return ef.replace(keys, reps, [seg], first, is_word)[0]
    if kind == "leftmost":
        return [(e, k) for _, e, k in ef.leftmost(keys, [seg], first, is_word)]
    full = ef.find_all(keys, [seg])
    if words:
        full = ef.whole_words([seg], full, ef.key_lengths(keys), is_word)
    return [(e, k) for _, e, k in full]


def make(A, R, form, n, fl, algo="auto"):
    kind, first, words = FORMS[form]
    ww = text(fl, WORDS) if words else False
    if kind == "replace":
        return R[first].ascii_case_insensitive_stream_batch(n, algo=algo, whole_words=ww)
    if kind == "leftmost":
        return A.ascii_case_insensitive_stream_batch(n, algo=algo, leftmost_first=first, leftmost_longest=not first, whole_words=ww)
    return A.ascii_case_insensitive_stream_batch(n, algo=algo, whole_words=ww)


def released(form, want, pos, T, kl):
    """the records of the whole text's answer a stream must have reported after consuming pos letters (and no other)"""
    kind, _, words = FORMS[form]
    if kind == "all":
        return [(e, k) for e, k in want if e < pos - words]
    return [(e, k) for e, k in want if e - kl[k] + 1 < pos - T - words]


def run(A, R, form, fl, segs, rng, T, chunk=None, algo="auto"):
    """every stream fed its segments chunk by chunk (random subsets of streams in random order, empty chunks among them),
    each segment closed by finish (by reset for plain find_all); after every feed the lag bound holds, and at the end
    every segment's output equals the definition"""
    kind, first, words = FORMS[form]
    n = len(segs)
    S = make(A, R, form, n, fl, algo)
    assert S.ascii_case_insensitive
    kl = ef.key_lengths(A._keys_letters)
    reps = A._reps
    wants = [[definition(form, A._keys_letters, reps, seg) for seg in ss] for ss in segs]
    at = [[0, 0] for _ in range(n)]                         # segment, letters fed
    got = [[] for _ in range(n)]
    while any(si < len(ss) for (si, _), ss in zip(at, segs)):
        live = [s for s in range(n) if at[s][0] < len(segs[s])]
        ids = [int(x) for x in rng.permutation(live)[:int(rng.integers(1, len(live) + 1))]]
        pieces = []
        for s in ids:
            si, off = at[s]
            k = chunk if chunk is not None else int(rng.choice([0, 1, max(T, 1), T + 1, 3 * T + 1, int(rng.integers(0, 12))]))
            pieces.append(segs[s][si][off:off + k])
            at[s][1] += len(pieces[-1])
        out = S.feed([text(fl, p) for p in pieces], ids=ids)
        for j, s in enumerate(ids):
            if kind == "replace":
                got[s] += [ord(c) for c in out[j]] if fl != "bytes" else list(out[j])
            pos = at[s][1]
            if kind != "replace":
                got[s] += [(e, k) for h, e, k in zip(out.hay_id.tolist(), out.end_index.tolist(), out.key_id.tolist()) if h == s]
                assert got[s] == released(form, wants[s][at[s][0]], pos, T, kl), (form, s, pos)
            else:
                assert got[s] == wants[s][at[s][0]][:len(got[s])], (form, s, pos)
            if pos == len(segs[s][at[s][0]]) and rng.integers(0, 3):
                if kind == "all" and not words:
                    S.reset([s])
                else:
                    fin = S.finish([s])
                    if kind == "replace":
                        got[s] += [ord(c) for c in fin[0]] if fl != "bytes" else list(fin[0])
                    else:
                        got[s] += list(zip(fin.end_index.tolist(), fin.key_id.tolist()))
                assert got[s] == wants[s][at[s][0]], (form, s)
                assert S.positions[s] == 0
                got[s] = []
                at[s] = [at[s][0] + 1, 0]
    return S


def prepare(fl, keys):
    A = build(fl, keys)
    A._keys_letters = keys
    A._reps = [[0x2A] * (i % 3) + [0x5F] for i in range(len(keys))]
    R = {first: A.replacer({text(fl, k): text(fl, r) for k, r in zip(keys, A._reps)}, leftmost_first=first)
         for first in (False, True)}
    return A, R


def fuzz(case, forms, rng, trials, n_streams=3, algo="auto"):
    fl = FLAVOUR[case]
    for _ in range(trials):
        keys = random_keys(case, rng)
        A, R = prepare(fl, keys)
        T = max(len(k) for k in keys) - 1
        segs = [[random_text(case, keys, rng, int(rng.integers(0, 30))) for _ in range(int(rng.integers(1, 3)))]
                for _ in range(n_streams)]
        for form in forms:
            run(A, R, form, fl, segs, rng, T, algo=algo)


# ------------------------------------------------------------------ CPU: the Python layer on the restatement
@pytest.mark.parametrize("case", ["bytes", "latin1", "wide", "mixed"])
def test_python_layer_on_the_restatement(monkeypatch, case):
    emul_stream_fold.install(monkeypatch)
    fuzz(case, list(FORMS), np.random.default_rng(len(case)), 4)


def named_cases():
    A, R = prepare("bytes", [list(b"ab"), list(b"AB"), list(b"Ab"), list(b"xyZ")])
    S = A.ascii_case_insensitive_stream_batch(2)
    m = S.feed([b"xa", b"X"])                                 # ab / AB / Ab across a seam, all three ids ascending
    assert len(m) == 0
    m = S.feed([b"Bq", b"Yz"])                               # a capital split by chunk boundaries on both sides
    assert list(zip(m.hay_id.tolist(), m.end_index.tolist(), m.key_id.tolist())) == [(0, 2, 0), (0, 2, 1), (0, 2, 2), (1, 2, 3)]
    S = R[False].ascii_case_insensitive_stream_batch(1)
    out = S.feed([b"xY"]) + S.finish()                          # held letters keep their case through finish
    assert b"".join(out) == b"xY"
    S = R[False].ascii_case_insensitive_stream_batch(1)
    assert b"".join(S.feed([b"pA"]) + S.feed([b"bxY"]) + S.finish()) == b"p_xY"


def test_named_cases(monkeypatch):
    emul_stream_fold.install(monkeypatch)
    named_cases()


def test_refusals_attributes_and_shared_argument_checks(monkeypatch):
    emul_streams.install(monkeypatch)
    emul_stream_leftmost.install(monkeypatch)
    emul_leftmost_first.install(monkeypatch)
    emul_stream_fold.install(monkeypatch)
    A, R = prepare("bytes", [list(b"ab")])
    for B in (A.stream_batch(1), A.stream_batch(1, leftmost_first=True), R[False].stream_batch(1)):
        assert B.ascii_case_insensitive is False
    assert A.ascii_case_insensitive_stream_batch(1).ascii_case_insensitive is True
    assert R[True].ascii_case_insensitive_stream_batch(1).ascii_case_insensitive is True
    for kw in ({"long": True}, {"ignore_white_space": True}):
        with pytest.raises(TypeError):
            A.ascii_case_insensitive_stream_batch(1, **kw)
    # the factories raise what stream_batch raises for the same arguments
    for args, kw in (((-1,), {}), ((1,), {"algo": "long"}), ((1,), {"algo": "x"}), ((1,), {"leftmost_longest": True, "leftmost_first": True}),
                     ((1,), {"whole_words": 3})):
        errs = []
        for f in (A.stream_batch, A.ascii_case_insensitive_stream_batch):
            with pytest.raises(Exception) as e:
                f(*args, **kw)
            errs.append((type(e.value), str(e.value)))
        assert errs[0] == errs[1], (args, kw)
    for args, kw in (((-1,), {}), ((1,), {"algo": "long"}), ((1,), {"whole_words": 3})):
        errs = []
        for f in (R[False].stream_batch, R[False].ascii_case_insensitive_stream_batch):
            with pytest.raises(Exception) as e:
                f(*args, **kw)
            errs.append((type(e.value), str(e.value)))
        assert errs[0] == errs[1], (args, kw)
    mod = pkg.flavour("unicode")
    Q = mod.Automaton(mod.STORE_INTS, mod.KEY_SEQUENCE)
    Q.add_word((1, 2), 0)
    Q.make_automaton()
    with pytest.raises(ValueError, match="KEY_SEQUENCE"):
        Q.ascii_case_insensitive_stream_batch(1)
    with pytest.raises(ValueError, match="KEY_SEQUENCE"):
        Q.replacer({(1, 2): (3,)}).ascii_case_insensitive_stream_batch(1)
    S = A.ascii_case_insensitive_stream_batch(1, leftmost_longest=True)
    P = R[False].ascii_case_insensitive_stream_batch(1)
    A.add_word(b"cd", 1)
    A.make_automaton()
    for call in (lambda: S.feed([b"ab"]), lambda: P.feed([b"ab"]), lambda: R[False].ascii_case_insensitive_stream_batch(1)):
        with pytest.raises(ValueError, match="changed"):
            call()
    with pytest.raises(ValueError, match="finish"):
        A.ascii_case_insensitive_stream_batch(1).finish()


def no_key():
    A = pkg.flavour("bytes").Automaton(pkg.flavour("bytes").STORE_INTS)
    A.add_word(b"x", 0)
    A.remove_word(b"x")
    A.make_automaton()
    assert A._fold_host(False) is None
    R = A.replacer({})
    S = A.ascii_case_insensitive_stream_batch(2, leftmost_first=True)
    assert len(S.feed([b"Ab", b"x"])) == 0 and len(S.finish()) == 0
    P = R.ascii_case_insensitive_stream_batch(1)
    assert b"".join(P.feed([b"Ab"]) + P.finish()) == b"Ab"


def test_no_key(monkeypatch):
    emul_stream_fold.install(monkeypatch)
    no_key()


# ------------------------------------------------------------------ the GPU
@pytest.mark.gpu
@pytest.mark.parametrize("algo", ["filter", "dfa"])
@pytest.mark.parametrize("case", ["bytes", "latin1", "wide", "mixed"])
def test_gpu_fuzz_against_the_definition(case, algo):
    fuzz(case, list(FORMS), np.random.default_rng(7 + len(case) + len(algo)), 6, n_streams=5, algo=algo)


@pytest.mark.gpu
def test_gpu_named_cases_and_no_key():
    named_cases()
    no_key()


def _flip(hays, rng):
    """the letters of hays with every ASCII letter's case flipped at random"""
    out = hays.copy()
    flip = rng.integers(0, 2, size=out.shape).astype(bool) & (((out | 0x20) >= 0x61) & ((out | 0x20) <= 0x7A))
    out[flip] ^= 0x20
    return out


def _collect(B, feeds, finish):
    """the rows of every feed (and finish) of B, in stream order then as delivered"""
    parts = [rows(B.feed(t)) for t in feeds] + ([rows(B.finish())] if finish else [])
    r = np.concatenate(parts) if parts else np.empty((0, 3), np.int64)
    return r[np.argsort(r[:, 0], kind="stable")]


def _replace_all(S, feeds, n):
    """the concatenated output of a replacing stream over CUDA tensor feeds and its finish: (flat bytes, offsets)"""
    per = [[] for _ in range(n)]
    for t in feeds:
        out, offs = S.feed(t)
        out, offs = out.cpu().numpy(), offs.cpu().numpy()
        for i in range(n):
            per[i].append(out[offs[i]:offs[i + 1]].tobytes())
    for i, x in enumerate(S.finish()):
        per[i].append(x)
    joined = [b"".join(p) for p in per]
    offs = np.zeros(n + 1, np.int64)
    np.cumsum([len(x) for x in joined], out=offs[1:])
    return np.frombuffer(b"".join(joined), np.uint8), offs


@pytest.mark.gpu
@pytest.mark.parametrize("swapped", [False, True])
@pytest.mark.parametrize("step", [256, 1, 7, 64])
def test_gpu_c2_million_streams(step, swapped):
    """10^6 streams of case-flipped C2 text fed `step` letters at a time, with C2's keys or with C2's keys and every key's
    swapcase() (aliases, also across seams); against the whole-batch case-insensitive methods on the whole rows.  At one
    letter per feed the staged forms (leftmost-longest, leftmost-first, replacing) run on the first 2^16 streams: each of
    their 256 feeds waits for the device three to four times, and what one-letter chunks exercise -- held letters carried
    through every feed, a match released letters after it ends -- happens in every stream alike; find_all runs all 10^6."""
    import torch
    from pyahocorasick_b200 import synth
    w = synth.make("C2")
    keys = list(w.keys)
    if swapped:
        have = set(keys)
        keys += [k.swapcase() for k in w.keys if k.swapcase() not in have]
    A = pkg.flavour("bytes").Automaton(pkg.flavour("bytes").STORE_INTS)
    for i, k in enumerate(keys):
        A.add_word(k, i)
    A.make_automaton()
    hay = _flip(w.haystacks, np.random.default_rng(step))
    n = hay.shape[0]
    d = torch.from_numpy(hay).cuda()
    feeds = [d[:, i:i + step].contiguous() for i in range(0, d.shape[1], step)]
    want_all = rows(A.find_all_batch(d, ascii_case_insensitive=True))
    assert np.array_equal(_collect(A.ascii_case_insensitive_stream_batch(n), feeds, False), want_all)
    if step == 1:
        n = 1 << 16
        d = d[:n]
        feeds = [t[:n] for t in feeds]
    for first in (False, True):
        want = rows((A.find_leftmost_first_batch if first else A.find_leftmost_longest_batch)(d, ascii_case_insensitive=True))
        B = A.ascii_case_insensitive_stream_batch(n, leftmost_first=first, leftmost_longest=not first)
        assert np.array_equal(_collect(B, feeds, True), want), first
    R = A.replacer({k: k[:2].upper() + b"#" for k in keys})
    wout, woffs = R.replace_batch(d, ascii_case_insensitive=True)
    out, offs = _replace_all(R.ascii_case_insensitive_stream_batch(n), feeds, n)
    assert np.array_equal(offs, woffs.cpu().numpy()) and np.array_equal(out, wout.cpu().numpy())


@pytest.mark.gpu
@pytest.mark.parametrize("klen", [64, 1000, 5000])
def test_gpu_long_keys(klen):
    rng = np.random.default_rng(klen)
    base = sorted({bytes(rng.choice(list(b"aAb "), size=int(rng.integers(1, klen + 1))).astype(np.uint8)) for _ in range(6)}
                  | {bytes(rng.choice(list(b"ab "), size=klen).astype(np.uint8))})
    keys = base + [k.swapcase() for k in base[:3] if k.swapcase() not in base]
    A = build("bytes", [list(k) for k in keys])
    texts = []
    for _ in range(5):
        t = b""
        while len(t) < 3 * klen:
            t += keys[int(rng.integers(0, len(keys)))].swapcase() if rng.integers(0, 2) else bytes(rng.choice(list(b"aB c"), size=5).astype(np.uint8))
        texts.append(t)
    n = len(texts)
    wants = {"all": rows(A.find_all_batch(texts, ascii_case_insensitive=True)),
             "words": rows(A.find_all_batch(texts, whole_words=b"ab", ascii_case_insensitive=True)),
             "ll": rows(A.find_leftmost_longest_batch(texts, ascii_case_insensitive=True)),
             "lf": rows(A.find_leftmost_first_batch(texts, whole_words=b"ab", ascii_case_insensitive=True))}
    assert len(wants["ll"]) > 0
    R = A.replacer({k: k[: len(k) // 3] for k in keys})
    wout = R.replace_batch(texts, ascii_case_insensitive=True)
    batches = {"all": A.ascii_case_insensitive_stream_batch(n), "words": A.ascii_case_insensitive_stream_batch(n, whole_words=b"ab"),
               "ll": A.ascii_case_insensitive_stream_batch(n, leftmost_longest=True),
               "lf": A.ascii_case_insensitive_stream_batch(n, leftmost_first=True, whole_words=b"ab")}
    S = R.ascii_case_insensitive_stream_batch(n)
    got = {k: [] for k in batches}
    pos, outs = [0] * n, [b""] * n
    while any(p < len(t) for p, t in zip(pos, texts)):
        chunks = []
        for s in range(n):
            k = int(rng.choice([1, klen - 1, klen, klen + 1, 3 * klen]))
            chunks.append(texts[s][pos[s]:pos[s] + k])
            pos[s] += k
        for k, B in batches.items():
            got[k].append(rows(B.feed(chunks)))
        outs = [a + b for a, b in zip(outs, S.feed(chunks))]
    for k, B in batches.items():
        if k != "all":
            got[k].append(rows(B.finish()))
        r = np.concatenate(got[k])
        assert np.array_equal(r[np.argsort(r[:, 0], kind="stable")], wants[k]), k
    assert [a + b for a, b in zip(outs, S.finish())] == wout


@pytest.mark.gpu
def test_gpu_staged_batch_past_2_gib():
    """two chunks of 1.1 GB each: the staged batch passes 2^31 bytes; planted keys in mixed case cross the feeds'
    boundary, half of them inside a word"""
    import torch
    n, size = 2, 1_100_000_000
    d = torch.full((n, size), 0x20, dtype=torch.uint8, device="cuda")
    where = torch.arange(1 << 20, size - 8, 1 << 20, device="cuda")
    for s in range(n):
        for j, b in enumerate(b"NeEdLe"):
            d[s, where + j + s] = b
        d[s, where[::2] + s + 6] = ord("S")
    A = build("bytes", [list(b"needle"), list(b"EED"), list(b"le "), list(b"NEEDLE")])
    want_ll = rows(A.find_leftmost_longest_batch(d, whole_words=True, ascii_case_insensitive=True))
    want_all = rows(A.find_all_batch(d, whole_words=True, ascii_case_insensitive=True))
    cut = (1 << 20) * 7 + 3
    feeds = [d[:, :cut].contiguous(), d[:, cut:].contiguous()]
    del d
    torch.cuda.empty_cache()
    B = A.ascii_case_insensitive_stream_batch(n, leftmost_longest=True, whole_words=True)
    assert len(want_ll) > 1000 and np.array_equal(_collect(B, feeds, True), want_ll)
    assert np.array_equal(_collect(A.ascii_case_insensitive_stream_batch(n, whole_words=True), feeds, True), want_all)


@pytest.mark.gpu
def test_gpu_unicode_letters_at_seams():
    """the 4-byte stream: U+0141 and U+1F641 (0x41 in their low byte) next to seams never fold, A-Z do"""
    keys = [[0x61, 0x141], [0x41, 0x1F641, 0x62], [0x141, 0x61], [0x1F661, 0x61]]
    A, R = prepare("unicode", keys)
    text_ = [0x41, 0x141, 0x61, 0x1F641, 0x42, 0x161, 0x41, 0x1F641, 0x62, 0x1F661, 0x41, 0x61, 0x141]
    for form in FORMS:
        for cut in range(1, len(text_)):
            run(A, R, form, "unicode", [[text_]], np.random.default_rng(cut), 2, chunk=cut)


@pytest.mark.gpu
def test_gpu_capacity_contract():
    """capacities 0, 1, n-1 and n on every feed entry of a folded batch, one where the unexpanded count fits and the
    expanded one does not: nothing is committed, and the same feed with room gives the answer"""
    import torch
    keys = [b"ab", b"AB", b"Ab", b"b", b"B", b"ca"]
    A = build("bytes", [list(k) for k in keys])
    R = A.replacer({k: k + b"!" for k in keys})
    chunks = [b"xaB aB b ab ", b"b CA ", b"zz ab", b" c"]
    prime = [b"a", b"", b"", b"x ab"]
    flat = np.frombuffer(b"".join(chunks), dtype=np.uint8).copy()
    offs = np.zeros(5, np.int64)
    np.cumsum([len(c) for c in chunks], out=offs[1:])
    L = N.lib()
    tb = A._table_for(0, False, True)
    stream = torch.cuda.current_stream().cuda_stream
    d = torch.from_numpy(flat.copy()).cuda()
    d_off = torch.from_numpy(offs).cuda()

    def fresh(kind):
        B = {"find_all": lambda: A.ascii_case_insensitive_stream_batch(4),
             "words": lambda: A.ascii_case_insensitive_stream_batch(4, whole_words=True),
             "leftmost": lambda: A.ascii_case_insensitive_stream_batch(4, leftmost_first=True),
             "replace": lambda: R.ascii_case_insensitive_stream_batch(4)}[kind]()
        B.feed(prime)
        return B

    def feed_args(B, cap, out, found, host):
        if host:
            return (B._ss, tb, N.ptr(flat), flat.size, N.ptr(offs), 4, 0, None)
        return (B._ss, tb, d.data_ptr(), flat.size, d_off.data_ptr(), 4, 0, None)

    for kind, host, dev in (("find_all", L.acb_streams_feed_host, L.acb_streams_feed_device),
                            ("words", L.acb_streams_feed_words_host, L.acb_streams_feed_words_device),
                            ("leftmost", L.acb_streams_feed_leftmost_host, L.acb_streams_feed_leftmost_device)):
        ref = fresh(kind).feed(chunks)
        n = len(ref)
        assert n > 3
        caps = [0, 1, n - 1, n]
        if kind == "find_all":
            caps.append(n - 2)                               # room for the representatives, not for their aliases
        for cap in caps:
            for on_host in (True, False):
                B = fresh(kind)
                before = list(B.positions)
                found = ctypes.c_int64(0)
                if on_host:
                    out = np.zeros(max(cap, 1), dtype=N.MATCH_DTYPE)
                    tail = (0, N.ptr(out), cap, ctypes.byref(found), 0) if kind != "find_all" else (N.ptr(out), cap, ctypes.byref(found), 0, 1)
                    rc = host(*feed_args(B, cap, out, found, True), *tail)
                    assert found.value == n and rc == (N.ACB_OK if cap >= n else N.ACB_EOVERFLOW), (kind, cap)
                else:
                    dout = torch.full((max(cap, 1), 3), -7, dtype=torch.int32, device="cuda")
                    cnt = torch.zeros(1, dtype=torch.int64, device="cuda")
                    tail = (0, dout.data_ptr(), cap, cnt.data_ptr(), stream, 0) if kind != "find_all" else \
                        (dout.data_ptr(), cap, cnt.data_ptr(), stream, 0)
                    assert dev(*feed_args(B, cap, None, None, False), *tail) == N.ACB_OK
                    assert int(cnt.item()) == n, (kind, cap)
                if cap >= n:
                    assert list(B.positions) != before
                    continue
                assert list(B.positions) == before, (kind, cap, on_host)      # nothing committed
                m = B.feed(chunks)
                assert rows(m).tolist() == rows(ref).tolist(), (kind, cap, on_host)
    ref_out = fresh("replace").feed(chunks)
    total = sum(len(x) for x in ref_out)
    r = R._replacer(tb, False, 0)
    for cap in (0, 1, total - 1, total):
        S = fresh("replace")
        oo = np.zeros(5, np.int64)
        t = ctypes.c_int64(0)
        buf = np.full(cap + 16, 0xEE, np.uint8)
        rc = L.acb_streams_replace_host(S._ss, r, tb, N.ptr(flat), flat.size, N.ptr(offs), 4, 0, None, 0, 0, N.ptr(oo), N.ptr(buf),
                                        cap, ctypes.byref(t))
        assert t.value == total and rc == (N.ACB_OK if cap == total else N.ACB_EOVERFLOW)
        if cap == total:
            assert buf[:total].tobytes() == b"".join(ref_out)
            continue
        assert list(S.positions) == [1, 0, 0, 4] and S.feed(chunks) == ref_out
        S = fresh("replace")
        dout = torch.full((cap + 16,), 0xEE, dtype=torch.uint8, device="cuda")
        doo = torch.zeros(5, dtype=torch.int64, device="cuda")
        tt = torch.zeros(1, dtype=torch.int64, device="cuda")
        assert L.acb_streams_replace_device(S._ss, r, tb, d.data_ptr(), flat.size, d_off.data_ptr(), 4, 0, None, 0, doo.data_ptr(),
                                            dout.data_ptr(), cap, tt.data_ptr(), stream, 0) == N.ACB_OK
        assert int(tt.item()) == total and list(S.positions) == [1, 0, 0, 4] and S.feed(chunks) == ref_out


@pytest.mark.gpu
def test_gpu_cuda_tensors_on_a_side_stream():
    """CUDA tensor feeds on a side stream, one of them misaligned; the caller's chunks are not written"""
    import torch
    rng = np.random.default_rng(21)
    keys = [list(b"ab"), list(b"AB"), list(b"ba"), list(b"aBa"), list(b"b")]
    A, R = prepare("bytes", keys)
    texts = [[int(x) for x in rng.choice(list(b"aAbB "), size=28)] for _ in range(300)]
    d = torch.from_numpy(np.array(texts, dtype=np.uint8)).cuda()
    W = 7
    zero = torch.zeros((1, W), dtype=torch.uint8, device="cuda")
    views = {"whole": lambda i: d[:, i * W:(i + 1) * W].contiguous(),
             "misaligned": lambda i: torch.cat([zero, d[:, i * W:(i + 1) * W]])[1:]}
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    for name, piece in views.items():
        batches = {form: make(A, R, form, len(texts), "bytes") for form in ("all", "all_words", "first", "longest_words")}
        got = {form: [[] for _ in texts] for form in batches}
        S = make(A, R, "replace_first", len(texts), "bytes")
        outs = []
        with torch.cuda.stream(side):
            for i in range(4):
                t = piece(i)
                if name == "misaligned":
                    assert t.data_ptr() % 16 != 0
                keep = t.clone()
                for form, B in batches.items():
                    m = B.feed(t)
                    for h, e, k in zip(m.hay_id.tolist(), m.end_index.tolist(), m.key_id.tolist()):
                        got[form][h].append((e, k))
                outs.append(S.feed(t))
                assert torch.equal(t, keep)                  # the fold never writes caller memory
            fins = {form: B.finish() for form, B in batches.items() if form != "all"}
            rest = S.finish()
        side.synchronize()
        for form, m in fins.items():
            for h, e, k in zip(m.hay_id.tolist(), m.end_index.tolist(), m.key_id.tolist()):
                got[form][h].append((e, k))
        for s, t in enumerate(texts):
            for form in batches:
                assert got[form][s] == definition(form, keys, A._reps, t), (name, form, s)
            out = b"".join(o.cpu().numpy()[f.cpu().numpy()[s]:f.cpu().numpy()[s + 1]].tobytes() for o, f in outs) + rest[s]
            assert list(out) == definition("replace_first", keys, A._reps, t), (name, s)


@pytest.mark.gpu
def test_gpu_interleaved_with_other_calls():
    """case-insensitive and case-sensitive stream batches and whole-batch calls, interleaved on one automaton"""
    rng = np.random.default_rng(33)
    keys = [b"ab", b"AB", b"abc", b"Bc", b"c a", b"a"]
    A = build("bytes", [list(k) for k in keys])
    texts = [bytes(rng.choice(list(b"aAbBcC "), size=90).astype(np.uint8)) for _ in range(50)]
    R = A.replacer({k: k.lower() * 2 for k in keys})
    F = A.ascii_case_insensitive_stream_batch(50)
    P = A.stream_batch(50)
    B = A.ascii_case_insensitive_stream_batch(50, leftmost_longest=True, whole_words=True)
    Q = A.stream_batch(50, leftmost_longest=True, whole_words=True)
    S = R.ascii_case_insensitive_stream_batch(50)
    T = R.stream_batch(50)
    whole = {"F": rows(A.find_all_batch(texts, ascii_case_insensitive=True)), "P": rows(A.find_all_batch(texts)),
             "B": rows(A.find_leftmost_longest_batch(texts, whole_words=True, ascii_case_insensitive=True)),
             "Q": rows(A.find_leftmost_longest_batch(texts, whole_words=True))}
    wout, pout = R.replace_batch(texts, ascii_case_insensitive=True), R.replace_batch(texts)
    got = {k: [] for k in whole}
    so, to = [b""] * 50, [b""] * 50
    for i in range(0, 90, 13):
        chunks = [t[i:i + 13] for t in texts]
        for k, X in (("F", F), ("P", P), ("B", B), ("Q", Q)):
            got[k].append(rows(X.feed(chunks)))
            assert np.array_equal(rows(A.find_all_batch(texts, ascii_case_insensitive=True)), whole["F"])
        so = [a + b for a, b in zip(so, S.feed(chunks))]
        assert R.replace_batch(texts) == pout
        to = [a + b for a, b in zip(to, T.feed(chunks))]
    got["B"].append(rows(B.finish()))
    got["Q"].append(rows(Q.finish()))
    for k in whole:
        r = np.concatenate(got[k])
        assert np.array_equal(r[np.argsort(r[:, 0], kind="stable")], whole[k]), k
    assert [a + b for a, b in zip(so, S.finish())] == wout
    assert [a + b for a, b in zip(to, T.finish())] == pout


@pytest.mark.gpu
def test_gpu_c_entries():
    A = build("bytes", [list(b"ab"), list(b"AB")])
    L = N.lib()
    plain = A._ensure_table(0)
    tb = A._table_for(0, False, True)
    ss = ctypes.c_void_p()
    assert L.acb_streams_new_folded(plain, 1, 0, N.SELECT_LONGEST, None, -1, ctypes.byref(ss)) == N.ACB_EINVAL
    for leftmost, kind, n_bits in ((0, 7, -1), (1, -1, -1), (2, N.SELECT_LONGEST, -1)):
        assert L.acb_streams_new_folded(tb, 1, leftmost, kind, None, -1, ctypes.byref(ss)) == N.ACB_EINVAL
    bits = np.zeros(1, np.uint32)
    assert L.acb_streams_new_folded(tb, 1, 1, N.SELECT_FIRST, N.ptr(bits), 1 << 40, ctypes.byref(ss)) == N.ACB_EINVAL
    assert L.acb_streams_new_folded(tb, -1, 0, N.SELECT_LONGEST, None, -1, ctypes.byref(ss)) == N.ACB_EINVAL
    flat = np.frombuffer(b"xaBx", dtype=np.uint8).copy()
    found = ctypes.c_int64()
    out = np.zeros(8, dtype=N.MATCH_DTYPE)
    F = A.ascii_case_insensitive_stream_batch(1)
    P = A.stream_batch(1)
    W = A.ascii_case_insensitive_stream_batch(1, whole_words=True)
    Lb = A.ascii_case_insensitive_stream_batch(1, leftmost_longest=True)
    assert L.acb_streams_feed_host(F._ss, plain, N.ptr(flat), 4, None, 1, 4, None, N.ptr(out), 8, ctypes.byref(found), 0, 1) == N.ACB_EINVAL
    assert L.acb_streams_feed_host(P._ss, tb, N.ptr(flat), 4, None, 1, 4, None, N.ptr(out), 8, ctypes.byref(found), 0, 1) == N.ACB_EINVAL
    for X in (W, Lb):
        feed = L.acb_streams_feed_words_host if X is W else L.acb_streams_feed_leftmost_host
        assert feed(X._ss, plain, N.ptr(flat), 4, None, 1, 4, None, 0, N.ptr(out), 8, ctypes.byref(found), 0) == N.ACB_EINVAL
    assert L.acb_streams_feed_host(F._ss, tb, N.ptr(flat), 4, None, 1, 4, None, N.ptr(out), 8, ctypes.byref(found), 0, 1) == N.ACB_OK
    assert found.value == 2 and out["key_id"][:2].tolist() == [0, 1]
    assert not P.positions.any() and F.positions.tolist() == [4]


@pytest.mark.gpu
def test_gpu_find_all_feed_refuses_a_stride_past_2_31_letters():
    """a chunk of 2^31 letters: its records could not say where they end, so the folded find_all feed refuses it with
    ACB_ERANGE before anything runs, as the plain feed does.  The check comes first, so no such buffer is needed."""
    import torch
    A = build("bytes", [list(b"ab"), list(b"AB")])
    L = N.lib()
    plain = A._ensure_table(0)                                 # first: a first upload of the plain table drops the others
    folded = A._table_for(0, False, True)
    stride = 1 << 31
    d = torch.zeros(64, dtype=torch.uint8, device="cuda")
    out = torch.zeros((4, 3), dtype=torch.int32, device="cuda")
    cnt = torch.zeros(1, dtype=torch.int64, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    for S, tb in ((A.ascii_case_insensitive_stream_batch(1), folded), (A.stream_batch(1), plain)):
        torch.cuda.synchronize()
        before = L.acb_launch_count()
        assert L.acb_streams_feed_device(S._ss, tb, d.data_ptr(), stride, None, 1, stride, None, out.data_ptr(), 4, cnt.data_ptr(),
                                         stream, 0) == N.ACB_ERANGE
        assert "2^31-1 letters" in N.last_error()
        assert L.acb_launch_count() == before and S.positions.tolist() == [0]


# launches of one feed: the fold before the scan; with case variants, the alias count and scatter (and, on a find_all
# word feed, nothing more: it already waits for its sizes)
FOLD, EXPAND = 1, 2


@pytest.mark.gpu
@pytest.mark.parametrize("variants", [False, True])
def test_gpu_launch_counts(variants):
    import torch
    keys = [b"ab", b"abc", b"bc"] + ([b"AB"] if variants else [])
    A = build("bytes", [list(k) for k in keys])
    R = A.replacer({k: b"X" for k in keys})
    chunks = [b"ab abc bc " * 3, b"abc ab"]
    d = torch.from_numpy(np.frombuffer(b"ab abc bc abc ab abc bc ", dtype=np.uint8).reshape(2, 12).copy()).cuda()
    L = N.lib()

    def count(B, x):
        B.feed([b"a", b"b"])
        before = L.acb_launch_count()
        B.feed(x)
        return L.acb_launch_count() - before

    for x in (chunks, d):
        plain = {"all": count(A.stream_batch(2), x=x), "words": count(A.stream_batch(2, whole_words=True), x=x),
                 "first": count(A.stream_batch(2, leftmost_first=True), x=x), "replace": count(R.stream_batch(2), x=x)}
        folded = {"all": count(A.ascii_case_insensitive_stream_batch(2), x=x),
                  "words": count(A.ascii_case_insensitive_stream_batch(2, whole_words=True), x=x),
                  "first": count(A.ascii_case_insensitive_stream_batch(2, leftmost_first=True), x=x),
                  "replace": count(R.ascii_case_insensitive_stream_batch(2), x=x)}
        extra = EXPAND if variants else 0
        assert folded == {"all": plain["all"] + FOLD + extra, "words": plain["words"] + FOLD + extra,
                          "first": plain["first"] + FOLD, "replace": plain["replace"] + FOLD}, x
