"""Every search route on million-key automata, against plain references that never call the library.

Three key sets, one alive at a time (class-scoped fixtures, freed on teardown), in this order:

* 800 k random 14-byte keys and the 10..13-byte prefixes of every 16th (256 classes, K * S past 2^31, MULTI anchors),
  STORE_INTS, built at the cost model's shape and forced onto the pair kernel and onto gram 4 / stride 4, then a
  65 MiB host batch on the pipelined route with keys at and beside its chunk cuts;
* the reference's published benchmark shape, bytes flavour: 1 M random words of 3..32 characters over [A-Za-z0-9],
  each stored with itself as value (14.7 M states, 63 classes; the filter saturates at gram 2 / stride 2, so every
  second letter starts a walk through a 3.7 GB goto table), searched in the published 1 M-character text with whole
  words planted every ~160 letters, two in three of 20..32 letters, so that walks reach deep states;
* the same words, unicode flavour: 58.9 M states (past 2^25) and a goto table of 3.8 G entries (past 2^31).  Latin-1
  text runs on its 1-byte table; text with a U+0142 every ~4 KiB and in every haystack runs on the wide table, where
  the gram is one letter, every probe passes and nearly every anchor entry is MULTI.  No key holds U+0142, so the
  reference is the bytes oracle over the same text with that letter replaced by a byte of no key.  ASCII case folding on
  the wide table is not tested here: it would build a second trie of tens of millions of states on top of the 40 GB
  the unicode set already holds on the host.  The planted words give thousands of matches of 16 letters or more, walks
  through states whose ids lie past 2^24.  The published words, their oracle and the shared references live from the
  first published group to the end of the module; the folded oracle is freed after the bytes group.

References: the C oracle's full list and iter_long, the reference extension's iter() where oracle/_ref is built,
batch_cases.np_greedy / first_cases.np_greedy_first for the leftmost rules, emul_replace / emul_words definitions, and
for ASCII folding the oracle over folded text and folded keys (one representative per group) with the aliases added by
emul_fold.expand.  Stream batches are compared with the reference over each stream's whole text and with the
whole-batch method.  A group whose host memory is not available is skipped with both numbers."""
import ctypes
import gc
import os
import string
import threading

import numpy as np
import pytest

import emul_fold
import oracle
import pyahocorasick_b200 as pkg
from batch_cases import np_greedy, published, rows
from emul_replace import definition as replaced
from emul_words import definition as whole_words
from first_cases import np_greedy_first
from pyahocorasick_b200 import _native as N

pytestmark = pytest.mark.gpu

N_WORDS = 1_000_000
N_HAY = 4096
WIDE = "ł"                        # in no key; forces the 4-byte table
NOT_KEY = ord("#")                     # in no key either: stands for WIDE in the reference text
SIZES = (1, 7, 31, 32, 33, 256)        # stream chunk sizes around T = longest word - 1 = 31
WORD = string.ascii_letters
GB = 1 << 30


# ------------------------------------------------------------------ host memory
def _mem_available():
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) << 10
    return 0


def _need(gb, what):
    have = _mem_available()
    if have < gb * GB:
        pytest.skip(f"{what} needs about {gb} GB of host memory; {have / GB:.1f} GB available")


class _PeakRss:
    """the largest resident set of this process while a group runs, sampled every 50 ms"""

    def __init__(self):
        self.peak = 0
        self._stop = threading.Event()
        self._t = threading.Thread(target=self._run, daemon=True)
        self._t.start()

    def _run(self):
        page = os.sysconf("SC_PAGE_SIZE")
        while True:
            with open("/proc/self/statm") as f:
                self.peak = max(self.peak, int(f.read().split()[1]) * page)
            if self._stop.wait(0.05):
                return

    def stop(self, what):
        self._stop.set()
        self._t.join()
        print(f"\n[large automata] {what}: peak host RSS {self.peak / GB:.1f} GiB")


def _device_bytes(A, tb, what):
    n = int(A._lib.acb_table_device_bytes(tb))
    print(f"\n[large automata] {what}: acb_table_device_bytes {n} ({n / GB:.2f} GiB)")
    return n


def _view(A):
    """states, classes and filter of the automaton's own trie, without copying its tables"""
    fv = N.FlatView()
    N.check(A._lib.acb_trie_flat_view(A._trie, ctypes.byref(fv)))
    return fv


# ------------------------------------------------------------------ batches and references
def _cuts(rng, n, n_hay):
    """int64 offsets of n_hay ragged haystacks over n letters, about 1 % of them empty"""
    pos = np.sort(rng.integers(0, n + 1, size=n_hay - 1))
    dup = rng.random(n_hay - 1) < 0.01
    pos[1:][dup[1:]] = pos[:-1][dup[1:]]
    return np.concatenate([[0], pos, [n]]).astype(np.int64)


def _split(buf, offs):
    return [buf[offs[i]:offs[i + 1]] for i in range(len(offs) - 1)]


def _ref(O, flat, offs):
    """the oracle's full list as int64 rows (hay, end, key id), in the reference's order"""
    return O.scan_batch_bytes(np.frombuffer(flat, np.uint8) if isinstance(flat, bytes) else flat, offs).astype(np.int64)


def _records(a):
    r = np.empty(len(a), dtype=N.MATCH_DTYPE)
    for j, f in enumerate(("hay_id", "end_index", "key_id")):
        r[f] = a[:, j]
    return r


def _longest(full, klen):
    return np_greedy(_records(full), klen)


def _first(full, klen):
    return np_greedy_first(_records(full), klen)


def _words_only(hays, full, klen, word_letters):
    """emul_words.definition over int64 rows; hays as bytes"""
    bits = set(word_letters)
    out = whole_words(hays, [tuple(r) for r in full.tolist()], klen, bits.__contains__)
    return np.array(out, dtype=np.int64).reshape(-1, 3)


def _replaced(hays, chosen, klen, reps):
    """emul_replace.definition per haystack -> bytes"""
    by_hay = [[] for _ in hays]
    for h, e, k in chosen.tolist():
        by_hay[h].append((e, k))
    return [bytes(replaced(h, c, klen, reps)) for h, c in zip(hays, by_hay)]


def _eq(got, want, what):
    got = np.asarray(got, dtype=np.int64).reshape(-1, 3)
    want = np.asarray(want, dtype=np.int64).reshape(-1, 3)
    if got.shape == want.shape and np.array_equal(got, want):
        return
    n = min(len(got), len(want))
    bad = np.nonzero((got[:n] != want[:n]).any(axis=1))[0]
    i = int(bad[0]) if len(bad) else n
    raise AssertionError(f"{what}: {len(got)} records, want {len(want)}; first difference at {i}: "
                         f"{got[i].tolist() if i < len(got) else None} vs {want[i].tolist() if i < len(want) else None}")


def _sorted(a):
    a = np.asarray(a, dtype=np.int64).reshape(-1, 3)
    return a[np.lexsort((a[:, 2], a[:, 1], a[:, 0]))]


class _Fold:
    """ASCII folding restated: representatives (the first id of every folded text, as emul_fold.groups), the alias
    lists (emul_fold.alias_csr's layout) and the oracle over the folded keys of the representatives"""

    def __init__(self, words_bytes):
        first = {}
        rep = np.empty(len(words_bytes), dtype=np.int64)
        for kid, k in enumerate(words_bytes):
            rep[kid] = first.setdefault(k.lower(), kid)
        self.rep = rep
        alias = np.nonzero(rep != np.arange(len(rep)))[0]
        cnt = np.bincount(rep[alias], minlength=len(rep) + 1)[:len(rep) + 1]
        self.ptr = np.concatenate([[0], np.cumsum(cnt)]).astype(np.int64)
        self.ids = alias[np.argsort(rep[alias], kind="stable")]
        self.sizes = np.bincount(rep)
        self.O = oracle.OracleAutomaton()
        for k, kid in first.items():
            self.O.add_word(k, kid)
        self.O.make_automaton()

    def scan(self, flat, offs):
        """(representatives only, expanded) rows of the folded text"""
        low = np.frombuffer(bytes(flat).lower(), np.uint8)
        reps = _ref(self.O, low, offs)
        full, total = emul_fold.expand(reps, self.ptr, self.ids, 1 << 62)
        assert len(full) == total
        return reps, full


def _feed_streams(sb, texts, sizes, finish=True, replace=False):
    """feed every stream its text in chunks of `sizes` (rotating, a different phase per stream) -> int64 rows sorted
    stably by stream (records), or the output per stream (replace)"""
    n = len(texts)
    pos = [0] * n
    got = [[] for _ in range(n)] if replace else []
    r = 0
    while any(p < len(t) for p, t in zip(pos, texts)):
        chunks = []
        for s, t in enumerate(texts):
            k = sizes[(r + s) % len(sizes)]
            chunks.append(t[pos[s]:pos[s] + k])
            pos[s] += k
        out = sb.feed(chunks)
        if replace:
            for s in range(n):
                got[s].append(out[s])
        else:
            got.append(rows(out))
        r += 1
    if not finish:                         # a find_all stream holds nothing back: finish() is refused
        with pytest.raises(ValueError, match="finish"):
            sb.finish()
    else:
        out = sb.finish()
        if replace:
            for s in range(n):
                got[s].append(out[s])
        else:
            got.append(rows(out))
    if replace:
        return [texts[0][:0].join(g) for g in got]
    a = np.concatenate(got) if got else np.empty((0, 3), np.int64)
    return a[np.argsort(a[:, 0], kind="stable")]


# ------------------------------------------------------------------ key set 3: 256 classes, MULTI anchors
def _k256_keys():
    rng = np.random.default_rng(5)
    raw = rng.integers(0, 256, size=(800_000, 14), dtype=np.uint8)
    keys = [bytes(r) for r in raw]
    keys += [keys[i][:10 + (i // 16) % 4] for i in range(0, len(raw), 16)]
    return list(dict.fromkeys(keys))


def _planted(rng, keys, n_bytes, n_hay, n_plant):
    """n_bytes random bytes with keys, prefixes and near misses (last byte changed, one byte short) planted 64 bytes
    apart, cut into n_hay ragged haystacks, some cuts through plants -> (flat, offsets, [(start, key)] of the planted keys)"""
    buf = rng.integers(0, 256, size=n_bytes, dtype=np.uint8)
    at = np.sort(rng.choice(n_bytes // 64 - 1, size=n_plant, replace=False)) * 64 + rng.integers(0, 40, size=n_plant)
    pick = rng.integers(0, len(keys), size=n_plant)
    kind = rng.integers(0, 4, size=n_plant)
    plants = []
    for p, k, how in zip(at.tolist(), pick.tolist(), kind.tolist()):
        w = keys[k]
        if how == 2:
            w = w[:-1] + bytes([(w[-1] + 1) % 256])
        elif how == 3:
            w = w[:-1]
        else:
            plants.append((p, k))
        buf[p:p + len(w)] = np.frombuffer(w, np.uint8)
    cuts = np.concatenate([rng.integers(0, n_bytes, size=n_hay // 2),
                           at[rng.integers(0, n_plant, size=n_hay // 2)] + rng.integers(1, 10, size=n_hay // 2)])
    offs = np.unique(np.concatenate([[0], np.clip(cuts, 0, n_bytes), [n_bytes]])).astype(np.int64)
    return buf, offs, plants


@pytest.fixture(scope="class")
def k256():
    _need(18, "the 256-class key set")
    peak = _PeakRss()
    keys = _k256_keys()
    O = oracle.OracleAutomaton()
    for i, k in enumerate(keys):
        O.add_word(k, i)
    O.make_automaton()
    rng = np.random.default_rng(21)
    flat, offs, _ = _planted(rng, keys, 4 << 20, 2048, 40_000)
    want = _ref(O, flat, offs)
    klen = np.fromiter(map(len, keys), dtype=np.int64, count=len(keys))
    d = dict(keys=keys, O=O, flat=flat, offs=offs, want=want, klen=klen, A=None)
    yield d
    peak.stop("key set 3 (256 classes)")
    d.clear()
    gc.collect()


def _k256_build(keys, mp, env):
    mod = pkg.flavour("bytes")
    A = mod.Automaton(mod.STORE_INTS)
    for i, k in enumerate(keys):
        A.add_word(k, i)
    with mp.context() as m:
        if env is None:
            m.delenv("ACB_FILTER", raising=False)
        else:
            m.setenv("ACB_FILTER", env)
        m.delenv("ACB_FORCE_TAGMAP", raising=False)
        A.make_automaton()
    return A


@pytest.mark.gpu
class TestK256:
    @pytest.mark.parametrize("env,shape", [("4,1,0,1", (4, 1, 2)), ("4,4,0,0", (4, 4, 1))])     # pair; single, wide
    def test_forced_shapes(self, k256, monkeypatch, env, shape):
        A = _k256_build(k256["keys"], monkeypatch, env)
        fs = A.filter_shape()
        assert (fs["gram_bytes"], fs["stride"], fs["filter_flags"]) == shape, fs
        for algo in ("filter", "dfa"):
            _eq(rows(A.find_all_batch((k256["flat"], k256["offs"]), algo=algo)), k256["want"], f"{env} {algo}")
        del A
        gc.collect()

    def test_default_shape(self, k256, monkeypatch):
        A = _k256_build(k256["keys"], monkeypatch, None)
        k256["A"] = A
        fv = _view(A)
        assert fv.n_classes == 256 and fv.n_states * fv.n_classes > 2 ** 31, (fv.n_states, fv.n_classes)
        fs = A.filter_shape()
        assert (fs["gram_bytes"], fs["stride"], fs["filter_flags"]) == (7, 4, 0), fs
        _device_bytes(A, A._ensure_table(0), "key set 3 table")
        flat, offs, O = k256["flat"], k256["offs"], k256["O"]
        for algo in ("filter", "dfa"):
            _eq(rows(A.find_all_batch((flat, offs), algo=algo)), k256["want"], algo)
        want = O.iter_long_batch_letters(oracle._letters(flat.tobytes()), offs)
        _eq(rows(A.find_long_batch((flat, offs))), want, "iter_long")
        _eq(rows(A.find_leftmost_longest_batch((flat, offs))), _longest(k256["want"], k256["klen"]), "longest")

    def test_stream_batch(self, k256):
        A = k256["A"]
        assert A is not None
        flat = k256["flat"][:1 << 20]
        so = _cuts(np.random.default_rng(22), flat.size, 256)
        texts = _split(flat.tobytes(), so)
        full = _ref(k256["O"], flat, so)
        _eq(_feed_streams(A.stream_batch(len(texts)), texts, (1, 7, 13, 14, 15, 256), False), full, "T = 13 stream")
        _eq(_feed_streams(A.stream_batch(len(texts), leftmost_longest=True), texts, (1, 7, 13, 14, 15, 256)),
            _longest(full, k256["klen"]), "T = 13 longest stream")

    def test_pipelined_64_mib(self, k256):
        """65 MiB of host text: the filter route uploads and scans it in 32 MiB chunks, chunk c scanning the start
        positions below c * 32 MiB - reach (reach: the longest key rounded up to 32 bytes); the DFA route scans it whole"""
        A, keys, O = k256["A"], k256["keys"], k256["O"]
        assert A is not None
        assert "ACB_NO_PIPELINE" not in os.environ, "the pipelined route is switched off"
        rng = np.random.default_rng(23)
        n = (64 << 20) + (1 << 20)
        base, _, plants = _planted(rng, keys, n, 2, 100_000)
        chunk = 32 << 20
        reach = (max(map(len, keys)) + 31) & ~31
        offs = np.unique(np.concatenate([[0], rng.integers(1, n, size=255), [n]])).astype(np.int64)
        offs = offs[~np.isin(offs, [chunk - reach + d for d in range(-40, 40)] + [2 * chunk - reach + d for d in range(-40, 40)])]
        windows = set(rng.integers(0, len(offs) - 1, size=40).tolist())
        for shift in (-1, 0, 1):
            buf = base.copy()
            # 14-byte keys starting one before, at and one after each start-position cut, and across each upload cut
            across = [(c * chunk - reach + shift, 2 * c + shift + 1) for c in (1, 2)] + [(chunk - 13, 7), (2 * chunk - 1, 8)]
            for p, k in across:
                buf[p:p + 14] = np.frombuffer(keys[k], np.uint8)
            live = [(p, k) for p, k in plants if bytes(buf[p:p + len(keys[k])]) == keys[k]] + across
            f = rows(A.find_all_batch((buf, offs), algo="filter"))
            if shift == 0:
                _eq(f, rows(A.find_all_batch((buf, offs), algo="dfa")), "filter vs dfa, 65 MiB")
            got = set(map(tuple, f.tolist()))
            for p, k in live:
                e = p + len(keys[k]) - 1
                h = int(np.searchsorted(offs, p, side="right")) - 1
                if offs[h + 1] > e:
                    assert (h, e - int(offs[h]), k) in got, (shift, p, k)
            near = {int(np.searchsorted(offs, p, side="right")) - 1 for p, _ in across}
            for h in sorted(near | (windows if shift == 0 else set())):
                a, b = int(offs[h]), int(offs[h + 1])
                want = _ref(O, buf[a:b], np.array([0, b - a], np.int64))
                want[:, 0] = h
                _eq(f[f[:, 0] == h], want, f"shift {shift}, window {h}")


# ------------------------------------------------------------------ the published data, shared by key sets 1 and 2
class _Published:
    """the published words (key id = generation order), the published text with whole words planted into it, its ragged
    cuts, wide variant and stream cuts, the bytes oracle and the references both flavours share"""

    def __init__(self):
        rng = np.random.default_rng(11)
        pw = published(N_WORDS, text_length=1_000_000)
        self.words = pw.words
        self.wb = [w.encode() for w in self.words]
        self.klen = np.fromiter(map(len, self.wb), dtype=np.int64, count=len(self.wb))
        # whole words every ~160 letters, two in three of 20..32 letters: random text alone rarely walks deeper than
        # six letters, and the unicode trie's state ids past 2^24 are those of nodes about seven letters deep
        t = np.frombuffer(pw.text.encode(), np.uint8).copy()
        n = t.size
        long_ids = np.nonzero(self.klen >= 20)[0]
        at = np.arange(0, n - 40, 160) + rng.integers(0, 120, size=len(range(0, n - 40, 160)))
        pick = np.where(rng.random(len(at)) < 2 / 3, rng.choice(long_ids, size=len(at)), rng.integers(0, N_WORDS, size=len(at)))
        for p, k in zip(at.tolist(), pick.tolist()):
            t[p:p + self.klen[k]] = np.frombuffer(self.wb[k], np.uint8)
        self.tb = t.tobytes()
        self.text = self.tb.decode()
        self.offs = _cuts(rng, n, N_HAY)
        self.hays = _split(self.tb, self.offs)
        # the wide text: U+0142 every 4 KiB and at the start of every non-empty haystack; '#' in the reference text
        starts = self.offs[:-1][np.diff(self.offs) > 0]
        spots = np.union1d(np.arange(0, n, 4096), starts)
        w = t.copy()
        w[spots] = NOT_KEY
        self.tb_w = w.tobytes()
        self.text_w = self.tb_w.decode("latin-1").replace("#", WIDE)
        self.hays_w = _split(self.tb_w, self.offs)
        self.streams = _cuts(np.random.default_rng(12), n, 1024)
        self.O = oracle.OracleAutomaton()
        for i, k in enumerate(self.wb):
            self.O.add_word(k, i)
        self.O.make_automaton()
        self._fold = None
        self._fold_scans = {}
        # references shared by both flavours
        self.full_text = _ref(self.O, self.tb, np.array([0, n], np.int64))
        self.full_ragged = _ref(self.O, self.tb, self.offs)
        self.full_text_w = _ref(self.O, self.tb_w, np.array([0, n], np.int64))
        self.full_ragged_w = _ref(self.O, self.tb_w, self.offs)
        rr = np.random.default_rng(13)
        lens = rr.integers(0, 41, size=len(self.wb))
        pool = rr.choice(np.frombuffer(b"abcdefghijklmnopqrstuvwxyz0123456789-_ .", np.uint8), size=int(lens.sum())).tobytes()
        ends = np.cumsum(lens).tolist()
        self.reps = [pool[e - k:e] for e, k in zip(ends, lens.tolist())]

    @property
    def fold(self):
        if self._fold is None:
            self._fold = _Fold(self.wb)
        return self._fold

    def fold_scan(self, offs):
        """_Fold.scan of the published text cut at offs, kept for later groups"""
        key = offs.tobytes()
        if key not in self._fold_scans:
            self._fold_scans[key] = self.fold.scan(np.frombuffer(self.tb, np.uint8), offs)
        return self._fold_scans[key]

    def release_fold(self):
        """free the folded oracle once key set 1 is done, keeping the ragged batch's answers key set 2 compares with"""
        self.fold_scan(self.offs)
        self._fold = None
        gc.collect()


@pytest.fixture(scope="module")
def pub():
    _need(6, "the published words and their oracle")
    p = _Published()
    yield p
    del p
    gc.collect()


# ------------------------------------------------------------------ key set 1: published, bytes flavour
@pytest.fixture(scope="class")
def bytes_set(pub):
    _need(13, "the published key set, bytes flavour, with its folded tables")
    peak = _PeakRss()
    mod = pkg.flavour("bytes")
    A = mod.Automaton(mod.STORE_ANY)
    for w in pub.wb:
        A.add_word(w, w)
    A.make_automaton()
    yield A
    pub.release_fold()
    peak.stop("key set 1 (published, bytes)")
    del A
    gc.collect()


@pytest.mark.gpu
class TestPublishedBytes:
    def test_shape_and_iter(self, pub, bytes_set):
        A = bytes_set
        fs = A.filter_shape()
        assert (fs["gram_bytes"], fs["stride"], fs["filter_flags"]) == (2, 2, 0), fs
        fv = _view(A)
        assert fv.n_keys == N_WORDS and fv.max_key_bytes == 32
        want = [(int(e), pub.wb[k]) for _, e, k in pub.full_text.tolist()]
        got = list(A.iter(pub.tb))
        assert got == want
        cb = []
        A.find_all(pub.tb, lambda e, v: cb.append((e, v)))
        assert cb == want
        _device_bytes(A, A._ensure_table(0), "key set 1 table")
        if oracle.ref_available("bytes"):
            R = oracle.ref_module("bytes").Automaton()
            for w in pub.wb:
                R.add_word(w, w)
            R.make_automaton()
            assert list(R.iter(pub.tb)) == got
            del R
            gc.collect()

    @pytest.mark.parametrize("algo", ["filter", "dfa"])
    def test_find_all_batch(self, pub, bytes_set, algo):
        A = bytes_set
        _eq(rows(A.find_all_batch([pub.tb], algo=algo)), pub.full_text, "one haystack")
        _eq(rows(A.find_all_batch(pub.hays, algo=algo)), pub.full_ragged, "ragged list")
        flat = np.frombuffer(pub.tb, np.uint8)
        _eq(rows(A.find_all_batch((flat, pub.offs), algo=algo)), pub.full_ragged, "ragged (flat, offsets)")
        _eq(_sorted(rows(A.find_all_batch((flat, pub.offs), algo=algo, sort=False))), _sorted(pub.full_ragged), "unsorted")
        import torch
        t = torch.from_numpy(flat.copy()).reshape(1000, 1000).cuda()
        want = _ref(pub.O, flat, np.arange(1001, dtype=np.int64) * 1000)
        _eq(rows(A.find_all_batch(t, algo=algo)), want, "CUDA tensor")

    def test_find_long_batch(self, pub, bytes_set):
        letters = oracle._letters(pub.tb)
        want = pub.O.iter_long_batch_letters(letters, pub.offs)
        _eq(rows(bytes_set.find_long_batch(pub.hays)), want, "iter_long per haystack")

    def test_leftmost(self, pub, bytes_set):
        A = bytes_set
        for algo in ("filter", "dfa"):
            _eq(rows(A.find_leftmost_longest_batch(pub.hays, algo=algo)), _longest(pub.full_ragged, pub.klen), "longest")
            _eq(rows(A.find_leftmost_first_batch(pub.hays, algo=algo)), _first(pub.full_ragged, pub.klen), "first")
        _eq(rows(A.find_leftmost_longest_batch([pub.tb])), _longest(pub.full_text, pub.klen), "longest, one haystack")

    def test_replacers(self, pub, bytes_set):
        A = bytes_set
        assert A.replacer().replace_batch(pub.hays) == pub.hays                  # each word replaced by itself
        mp = dict(zip(pub.wb, pub.reps))
        for first, sel in ((False, _longest), (True, _first)):
            R = A.replacer(mp, leftmost_first=first)
            assert R.replace_batch(pub.hays) == _replaced(pub.hays, sel(pub.full_ragged, pub.klen), pub.klen, pub.reps), first
            assert R.replace_batch([pub.tb]) == _replaced([pub.tb], sel(pub.full_text, pub.klen), pub.klen, pub.reps), first

    def test_whole_words(self, pub, bytes_set):
        A = bytes_set
        wl = WORD.encode()
        ww = _words_only(pub.hays, pub.full_ragged, pub.klen, wl)
        assert 0 < len(ww) < len(pub.full_ragged)
        _eq(rows(A.find_all_batch(pub.hays, whole_words=wl)), ww, "find_all whole words")
        _eq(rows(A.find_leftmost_longest_batch(pub.hays, whole_words=wl)), _longest(ww, pub.klen), "longest whole words")
        _eq(rows(A.find_leftmost_first_batch(pub.hays, whole_words=wl)), _first(ww, pub.klen), "first whole words")
        R = A.replacer(dict(zip(pub.wb, pub.reps)))
        assert R.replace_batch(pub.hays, whole_words=wl) == _replaced(pub.hays, _longest(ww, pub.klen), pub.klen, pub.reps)

    def test_ascii_case_insensitive(self, pub, bytes_set):
        A = bytes_set
        f = pub.fold
        assert f.sizes.max() >= 4 and (f.sizes >= 4).sum() > 10, np.bincount(f.sizes)
        reps, full = pub.fold_scan(pub.offs)
        assert len(full) > len(reps) > len(pub.full_ragged)
        _eq(rows(A.find_all_batch(pub.hays, ascii_case_insensitive=True)), full, "folded find_all")
        _eq(rows(A.find_leftmost_longest_batch(pub.hays, ascii_case_insensitive=True)), _longest(reps, pub.klen), "folded longest")
        _eq(rows(A.find_leftmost_first_batch(pub.hays, ascii_case_insensitive=True)), _first(reps, pub.klen), "folded first")
        R = A.replacer(dict(zip(pub.wb, pub.reps)))
        assert R.replace_batch(pub.hays, ascii_case_insensitive=True) == _replaced(pub.hays, _longest(reps, pub.klen), pub.klen, pub.reps)
        _device_bytes(A, A._table_for(0, False, True), "key set 1 folded table")

    def test_stream_batches(self, pub, bytes_set):
        A = bytes_set
        so = pub.streams
        texts = _split(pub.tb, so)
        full = _ref(pub.O, pub.tb, so)
        wl = WORD.encode()
        ww = _words_only(texts, full, pub.klen, wl)
        reps, ffull = pub.fold_scan(so)
        n = len(texts)
        cases = [
            ("find_all", dict(), False, full, lambda: A.find_all_batch(texts)),
            ("longest", dict(leftmost_longest=True), True, _longest(full, pub.klen), lambda: A.find_leftmost_longest_batch(texts)),
            ("first", dict(leftmost_first=True), True, _first(full, pub.klen), lambda: A.find_leftmost_first_batch(texts)),
            ("words", dict(whole_words=wl), True, ww, lambda: A.find_all_batch(texts, whole_words=wl)),
            ("words longest", dict(whole_words=wl, leftmost_longest=True), True, _longest(ww, pub.klen),
             lambda: A.find_leftmost_longest_batch(texts, whole_words=wl)),
            ("words first", dict(whole_words=wl, leftmost_first=True), True, _first(ww, pub.klen),
             lambda: A.find_leftmost_first_batch(texts, whole_words=wl)),
        ]
        for name, kw, fin, want, whole in cases:
            _eq(rows(whole()), want, name + " whole batch")
            _eq(_feed_streams(A.stream_batch(n, **kw), texts, SIZES, fin), want, name + " stream")
        fcases = [
            ("folded find_all", dict(), False, ffull),
            ("folded longest", dict(leftmost_longest=True), True, _longest(reps, pub.klen)),
            ("folded first", dict(leftmost_first=True), True, _first(reps, pub.klen)),
        ]
        for name, kw, fin, want in fcases:
            _eq(_feed_streams(A.ascii_case_insensitive_stream_batch(n, **kw), texts, SIZES, fin), want, name + " stream")
        R = A.replacer(dict(zip(pub.wb, pub.reps)))
        want = _replaced(texts, _longest(full, pub.klen), pub.klen, pub.reps)
        assert R.replace_batch(texts) == want
        assert _feed_streams(R.stream_batch(n), texts, SIZES, replace=True) == want
        want = _replaced(texts, _longest(reps, pub.klen), pub.klen, pub.reps)
        assert _feed_streams(R.ascii_case_insensitive_stream_batch(n), texts, SIZES, replace=True) == want


# ------------------------------------------------------------------ key set 2: published, unicode flavour
@pytest.fixture(scope="class")
def unicode_set(pub):
    _need(32, "the published key set, unicode flavour, with its latin-1 table")
    peak = _PeakRss()
    mod = pkg.flavour("unicode")
    A = mod.Automaton(mod.STORE_ANY)
    for w in pub.words:
        A.add_word(w, w)
    A.make_automaton()
    yield A
    peak.stop("key set 2 (published, unicode)")
    del A
    gc.collect()


@pytest.mark.gpu
class TestPublishedUnicode:
    def test_shape(self, unicode_set):
        A = unicode_set
        fv = _view(A)
        assert fv.n_states > 2 ** 25 and fv.n_states * fv.n_classes > 2 ** 31, (fv.n_states, fv.n_classes)
        fs = A.filter_shape()
        assert fs["filter_flags"] == 1 and fs["gram_bytes"] == 4, fs              # single placement, wide

    def test_latin1_text(self, pub, unicode_set):
        A = unicode_set
        got = list(A.iter(pub.text))
        assert got == [(int(e), pub.words[k]) for _, e, k in pub.full_text.tolist()]
        hays = [h.decode() for h in pub.hays]
        for algo in ("filter", "dfa"):
            _eq(rows(A.find_all_batch(hays, algo=algo)), pub.full_ragged, algo)
        assert A._narrow_table is not None
        _device_bytes(A, A._narrow_table, "key set 2 latin-1 table")
        _eq(rows(A.find_leftmost_longest_batch(hays)), _longest(pub.full_ragged, pub.klen), "longest")
        _eq(rows(A.find_leftmost_first_batch(hays)), _first(pub.full_ragged, pub.klen), "first")

    def test_latin1_ascii_case_insensitive(self, pub, unicode_set):
        hays = [h.decode() for h in pub.hays]
        _, full = pub.fold_scan(pub.offs)
        _eq(rows(unicode_set.find_all_batch(hays, ascii_case_insensitive=True)), full, "folded latin-1")

    @pytest.mark.parametrize("algo", ["filter", "dfa"])
    def test_wide_find_all(self, pub, unicode_set, algo):
        A = unicode_set
        hays = [h.decode("latin-1").replace("#", WIDE) for h in pub.hays_w]
        assert all(WIDE in h for h in hays if h)
        deep = int((pub.klen[pub.full_text_w[:, 2]] >= 16).sum())
        assert deep >= 2000, deep                  # walks that reach the trie's deep states, ids past 2^24
        _eq(rows(A.find_all_batch([pub.text_w], algo=algo)), pub.full_text_w, "wide, one haystack")
        _eq(rows(A.find_all_batch(hays, algo=algo)), pub.full_ragged_w, "wide, ragged")
        _eq(rows(A.find_leftmost_longest_batch(hays, algo=algo)), _longest(pub.full_ragged_w, pub.klen), "wide longest")
        _eq(rows(A.find_leftmost_first_batch(hays, algo=algo)), _first(pub.full_ragged_w, pub.klen), "wide first")

    def test_wide_iter_and_long(self, pub, unicode_set):
        A = unicode_set
        assert list(A.iter(pub.text_w)) == [(int(e), pub.words[k]) for _, e, k in pub.full_text_w.tolist()]
        _device_bytes(A, A._ensure_table(0), "key set 2 wide table")
        hays = [h.decode("latin-1").replace("#", WIDE) for h in pub.hays_w]
        want = pub.O.iter_long_batch_letters(oracle._letters(pub.tb_w), pub.offs)
        _eq(rows(A.find_long_batch(hays)), want, "wide iter_long")

    def test_wide_replacers_and_words(self, pub, unicode_set):
        A = unicode_set
        hays = [h.decode("latin-1").replace("#", WIDE) for h in pub.hays_w]
        assert A.replacer().replace_batch(hays) == hays
        mp = dict(zip(pub.words, (r.decode() for r in pub.reps)))
        for first, sel in ((False, _longest), (True, _first)):
            want = _replaced(pub.hays_w, sel(pub.full_ragged_w, pub.klen), pub.klen, pub.reps)
            got = A.replacer(mp, leftmost_first=first).replace_batch(hays)
            assert got == [w.decode("latin-1").replace("#", WIDE) for w in want], first
        ww = _words_only(pub.hays_w, pub.full_ragged_w, pub.klen, WORD.encode())
        _eq(rows(A.find_all_batch(hays, whole_words=WORD)), ww, "wide whole words")
        _eq(rows(A.find_leftmost_longest_batch(hays, whole_words=WORD)), _longest(ww, pub.klen), "wide whole-word longest")
        _eq(rows(A.find_leftmost_first_batch(hays, whole_words=WORD)), _first(ww, pub.klen), "wide whole-word first")

    def test_wide_stream_batches(self, pub, unicode_set):
        A = unicode_set
        so = pub.streams
        tb = _split(pub.tb_w, so)
        texts = [t.decode("latin-1").replace("#", WIDE) for t in tb]
        full = _ref(pub.O, pub.tb_w, so)
        ww = _words_only(tb, full, pub.klen, WORD.encode())
        n = len(texts)
        for name, kw, fin, want in (("find_all", dict(), False, full),
                                    ("longest", dict(leftmost_longest=True), True, _longest(full, pub.klen)),
                                    ("first", dict(leftmost_first=True), True, _first(full, pub.klen)),
                                    ("words", dict(whole_words=WORD), True, ww),
                                    ("words first", dict(whole_words=WORD, leftmost_first=True), True, _first(ww, pub.klen))):
            _eq(_feed_streams(A.stream_batch(n, **kw), texts, SIZES, fin), want, name + " stream")
        R = A.replacer(dict(zip(pub.words, (r.decode() for r in pub.reps))))
        want = [w.decode("latin-1").replace("#", WIDE) for w in _replaced(tb, _longest(full, pub.klen), pub.klen, pub.reps)]
        assert R.replace_batch(texts) == want
        assert _feed_streams(R.stream_batch(n), texts, SIZES, replace=True) == want
