"""Threads and devices: results that keep the values of the key set they were computed on, automata searched from several
threads at once, and a second GPU.

The native calls release the GIL, so threads overlap on the GPU; one automaton is serialised by its lock, different
automata run side by side in their own scratch.  Every answer here comes from a plain reference: the C oracle's full
list, emul_leftmost.greedy, first_cases (Python's re), emul_replace.definition, emul_words.definition, and the per-key
methods for the lookups.

A. Results are snapshots: Matches, stream feeds and the lookup lists give, after remove_word, pop, a new value, a new
   key or clear, what they gave right after the call.  On the CPU through the emulations, and on the GPU.
B. Threads on one GPU: independent automata over different kernels and table sizes at once; one automaton searched by
   several threads while another changes its key set; the first shared-memory opt-in of one kernel from several threads
   at once (a fresh process); unsynchronised CUDA outputs whose automaton changes or goes away while they are computed.
C. Two GPUs (skipped with fewer): the caller's current device is the same after every entry point, every feature gives
   the reference answer on device 1, one automaton moves between the devices, a thread per device, and scan_sharded
   over NCCL.

Every thread is joined and every spawned process joined with a timeout, terminated if still alive.  Each test runs its
interleaving once: nothing here repeats a scan to make a race happen."""
import gc
import multiprocessing
import os
import sys
import threading
import traceback

import numpy as np
import pytest

import emul
import emul_leftmost
import emul_leftmost_first
import emul_lookup
import emul_replace
import emul_select
import emul_streams
import emul_words
import first_cases
import kernel_cells
import oracle
import pyahocorasick_b200 as pkg
from batch_cases import forms, triples

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
MiB = 1 << 20
JOIN_S = 600                       # a thread or process still running after this has hung


def _device_count():
    try:
        import torch
        return torch.cuda.device_count() if torch.cuda.is_available() else 0
    except Exception:
        return 0


two_gpus = pytest.mark.skipif(_device_count() < 2, reason=f"needs 2 CUDA devices, this machine has {_device_count()}")


def _run_threads(targets, timeout=JOIN_S):
    """Start one thread per callable, all released together at a barrier; join every one.  Returns their results in
    order; re-raises the first exception with its traceback."""
    barrier = threading.Barrier(len(targets))
    out = [None] * len(targets)
    errors = []

    def body(i, f):
        try:
            barrier.wait(timeout=timeout)
            out[i] = f()
        except BaseException:                                   # reported below, with the thread's traceback
            errors.append((i, traceback.format_exc()))

    ts = [threading.Thread(target=body, args=(i, f), daemon=True) for i, f in enumerate(targets)]
    for t in ts:
        t.start()
    for t in ts:
        t.join(timeout)
    alive = [i for i, t in enumerate(ts) if t.is_alive()]
    assert not alive, f"threads {alive} still running after {timeout} s"
    assert not errors, "\n".join(f"thread {i}:\n{tb}" for i, tb in errors)
    return out


# ====================================================================== A. results are snapshots
STORES = {"ints": pkg.STORE_INTS, "length": pkg.STORE_LENGTH, "any": pkg.STORE_ANY}
CHANGES = ("remove_word", "pop", "new_value", "add_and_build", "clear")
SNAP_KEYS = ["he", "she", "his", "hers", "zero", "s", "中文"]
SNAP_HAYS = ["ushers zero his", "hershe", "", "s中文he hers"]


def _snap_setup(fl, store):
    """(A, model) over SNAP_KEYS: model = key -> (id, value) as added; STORE_INTS gives the first key the value 0"""
    mod = pkg.flavour(fl)
    A = mod.Automaton(STORES[store])
    keys = [k.encode() for k in SNAP_KEYS if k.isascii()] if fl == "bytes" else list(SNAP_KEYS)
    model = {}
    for i, k in enumerate(keys):
        if store == "length":
            A.add_word(k)
            v = len(k)
        else:
            v = 7 * i if store == "ints" else ("value", i)       # ints: key 0 has the value 0
            A.add_word(k, v)
        model[k] = (i, v)
    A.make_automaton()
    hays = [h.encode() if fl == "bytes" else h for h in SNAP_HAYS if fl != "bytes" or h.isascii()]
    return A, keys, hays, model


def _letters(x):
    return list(x) if isinstance(x, bytes) else [ord(c) for c in x]


def _snap_reference(fl, keys, hays, model):
    """every snapshot result as the references compute it for the key set `model`"""
    O = oracle.OracleAutomaton()
    for i, k in enumerate(keys):
        O.add_word(k, i)
    O.make_automaton()
    val = {i: v for i, v in model.values()}
    key_len = np.array([len(k) for k in keys])
    full = [(h, e, k) for h, t in enumerate(hays) for e, k in O.find_all(t)]
    case = "bytes" if fl == "bytes" else "wide"
    first = first_cases.find(case, [_letters(k) for k in keys], [_letters(h) for h in hays])
    return {
        "find_all": [(h, e, val[k]) for h, e, k in full],
        "long": [(h, e, val[k]) for h, t in enumerate(hays) for e, k in O.iter_long(t)],
        "leftmost_longest": [(h, e, val[k]) for h, e, k in emul_leftmost.greedy(full, key_len)],
        "leftmost_first": [(h, e, val[k]) for h, e, k in first],
    }


@pytest.mark.parametrize("change", CHANGES)
@pytest.mark.parametrize("store", list(STORES))
@pytest.mark.parametrize("fl", ["bytes", "unicode"])
def test_results_are_snapshots_emulated(fl, store, change, monkeypatch):
    emul.install(monkeypatch)
    emul_leftmost.install(monkeypatch)
    emul_streams.install(monkeypatch)
    emul_lookup.install(monkeypatch)
    emul_select.install(monkeypatch)
    emul_leftmost_first.install(monkeypatch)
    _check_live_snapshots(fl, store, change)


@pytest.mark.gpu
@pytest.mark.parametrize("change", CHANGES)
@pytest.mark.parametrize("store", list(STORES))
@pytest.mark.parametrize("fl", ["bytes", "unicode"])
def test_results_are_snapshots_gpu(fl, store, change):
    _check_live_snapshots(fl, store, change, cuda=True)


def _check_live_snapshots(fl, store, change, cuda=False):
    """Matches, stream feeds and lookup lists, asked again after the key set changed, give what they gave right after
    the call -- which is the reference of the key set at call time."""
    A, keys, hays, model = _snap_setup(fl, store)
    n = len(hays)
    want = _snap_reference(fl, keys, hays, model)
    res = {
        "find_all": A.find_all_batch(hays),
        "long": A.find_long_batch(hays),
        "leftmost_longest": A.find_leftmost_longest_batch(hays),
        "leftmost_first": A.find_leftmost_first_batch(hays),
        "stream_feed": A.stream_batch(n).feed(hays),
    }
    S = A.stream_batch(n, leftmost_first=True)
    res["first_feed"] = S.feed(hays)
    res["first_finish"] = S.finish()
    if cuda and fl == "bytes":
        import torch
        width = max(map(len, hays))
        rows = np.zeros((n, width), dtype=np.uint8)              # zero padding: no key holds a 0 byte
        for i, h in enumerate(hays):
            rows[i, :len(h)] = np.frombuffer(h, dtype=np.uint8)
        t = torch.from_numpy(rows).cuda()
        res["find_all_cuda"] = A.find_all_batch(t)
        res["leftmost_first_cuda"] = A.find_leftmost_first_batch(t)
    probe = keys + [keys[0] + keys[0][:1]]
    prefix = [keys[0][:1], keys[1][:1]]
    lists = {"get_batch": A.get_batch(probe, "missing"), "values_batch": A.values_batch(prefix),
             "items_batch": A.items_batch(prefix)}
    lists_want = {"get_batch": [model[k][1] if k in model else "missing" for k in probe],
                  "values_batch": [list(A.values(p)) for p in prefix],
                  "items_batch": [list(A.items(p)) for p in prefix]}
    refs = dict(want, stream_feed=want["find_all"], find_all_cuda=want["find_all"],
                leftmost_first_cuda=want["leftmost_first"])

    def per_hay(rows_):
        out = [[] for _ in range(n)]
        for h, e, v in rows_:
            out[h].append((e, v))
        return out

    def check(when):
        for name, m in res.items():
            if name in ("first_feed", "first_finish"):
                continue
            w = refs[name]
            assert list(m) == w, (name, when)
            assert m.values() == [v for _, _, v in w], (name, when)
            assert m.per_haystack(n) == per_hay(w), (name, when)
        both = list(res["first_feed"]) + list(res["first_finish"])
        assert sorted(both) == sorted(want["leftmost_first"]), when
        assert res["first_feed"].values() + res["first_finish"].values() == [v for _, _, v in both], when
        assert lists == lists_want, when

    check("right after the calls")
    k0 = keys[0]                                                 # a key with matches; STORE_INTS: the value 0
    assert model[k0][1] == (0 if store == "ints" else model[k0][1])
    if change == "remove_word":
        assert A.remove_word(k0)
    elif change == "pop":
        assert A.pop(k0) == model[k0][1]
    elif change == "new_value":
        if store == "length":
            A.add_word(k0)
        else:
            A.add_word(k0, 99 if store == "ints" else ("new", 0))
    elif change == "add_and_build":
        new = hays[0][:4]
        if store == "length":
            A.add_word(new)
        else:
            A.add_word(new, 5 if store == "ints" else ("new", 1))
        A.make_automaton()
    else:
        A.clear()
    check(f"after {change}")


# ====================================================================== B. threads on one GPU
def _obj(L, letters):
    return bytes(letters) if L == 1 else "".join(map(chr, letters))


class Job:
    """One automaton, its key set (letter tuples, key id = index = value), the oracle over it, and the fixed mixed
    sequence of calls a thread runs on it (run), each checked against a plain reference."""

    def __init__(self, A, keys, L, seed, fold=False):
        self.A, self.keys, self.L, self.fold = A, keys, L, fold
        self.rng = np.random.default_rng(seed)
        self.key_len = np.array([len(k) for k in keys])
        self.case = "bytes" if L == 1 else "wide"
        self.O = self._oracle([_obj(L, k) if L == 1 else tuple(k) for k in keys])
        self.alpha = sorted({x for k in keys for x in k})

    @staticmethod
    def _oracle(keys):
        O = oracle.OracleAutomaton()
        for i, k in enumerate(keys):
            O.add_word(k, i)
        O.make_automaton()
        return O

    def text(self, n_hay, max_len):
        """haystacks (letter lists) in the key alphabet with keys planted, one empty"""
        hays = []
        for i in range(n_hay):
            h = [int(x) for x in self.rng.choice(self.alpha, size=int(self.rng.integers(0, max_len)))]
            k = self.keys[int(self.rng.integers(0, len(self.keys)))]
            at = int(self.rng.integers(0, len(h) + 1))
            hays.append(h[:at] + list(k) + h[at:] if i else [])
        return hays

    def full(self, hays):
        """[(hay, end, key id)] in the reference's order; with fold, every key whose folded text occurs"""
        if not self.fold:
            return [(h, e, k) for h, t in enumerate(hays) for e, k in self.O.find_all(_obj(self.L, t))]
        fk = {}
        for i, k in enumerate(self.keys):
            fk.setdefault(bytes(k).lower(), []).append(i)
        Of = self._oracle(list(fk))
        groups = list(fk.values())
        out = []
        for h, t in enumerate(hays):
            for e, g in Of.find_all(bytes(t).lower()):
                out += [(h, e, k) for k in groups[g]]
        return sorted(out, key=lambda r: (r[0], r[1], -self.key_len[r[2]], r[2]))

    def big(self, n_bytes):
        """n_bytes of filler no key holds with a key planted every 4093 letters, cut raggedly (a cut at 32 MiB, where
        the host route pipelines): (flat bytes, byte offsets), and the reference records"""
        L = self.L
        n = n_bytes // L
        letters = np.full(n, 0x23 if L == 1 else 0x2603, dtype=np.uint8 if L == 1 else np.uint32)
        for i, b in enumerate(range(100, n - 200, 4093)):
            k = self.keys[i % len(self.keys)]
            letters[b:b + len(k)] = k
        cuts = np.sort(self.rng.integers(0, n, size=400))
        off = np.sort(np.concatenate([[0, 0], cuts, [32 * MiB // L] * 2, [n]])).astype(np.int64)
        flat = letters if L == 1 else letters.astype("<u4").view(np.uint8)
        if self.fold:
            want = None
        elif L == 1:
            want = [tuple(r) for r in self.O.scan_batch_bytes(flat, off).tolist()]
        else:
            want = [tuple(r) for r in self.O.scan_batch_letters(letters, off)]
        return (flat, off * L), want

    def run(self, device=None):
        """The fixed mixed sequence; device: the device every call names (None: the current one)"""
        import torch
        A, L, kw = self.A, self.L, {} if device is None else {"device": device}
        fold = {"ascii_case_insensitive": True} if self.fold else {}
        hays = self.text(40, 300)
        objs = [_obj(L, h) for h in hays]
        if self.fold:                                            # text in both cases
            objs = [o.upper() if i % 2 else o for i, o in enumerate(objs)]
            hays = [list(o) for o in objs]
        full = self.full(hays)
        for name, batch in forms(objs, hays, L, False):
            assert triples(A.find_all_batch(batch, **kw, **fold)) == full, name
        if not self.fold:
            assert [(h, e, k) for h, o in enumerate(objs) for e, k in A.find_long_batch(objs, **kw).per_haystack(len(objs))[h]] == \
                [(h, e, k) for h, o in enumerate(objs) for e, k in self.O.iter_long(o)]
        batch, want = self.big(48 * MiB)
        got = A.find_all_batch(batch, **kw, **fold)
        if want is not None:
            assert len(got) == len(want) and triples(got) == want
        else:
            assert len(got) > 0
        # a CUDA tensor on this thread's own stream
        dev = torch.cuda.current_device() if device is None else device
        rows = self.text(64, 200)
        width = max(map(len, rows))
        rows = [r + [0x20] * (width - len(r)) for r in rows]           # space padding: no key holds a space
        arr = np.asarray(rows, dtype=np.uint8 if L == 1 else "<u4").view(np.uint8).reshape(len(rows), -1)
        t = torch.from_numpy(arr).to(f"cuda:{dev}")
        if device is None:                                       # this thread's own stream
            with torch.cuda.stream(torch.cuda.Stream()):
                got = triples(A.find_all_batch(t, **fold))
                ll = triples(A.find_leftmost_longest_batch(t, **fold))
        else:                                                    # a tensor on `device`, whatever the current one is
            got = triples(A.find_all_batch(t, **fold))
            ll = triples(A.find_leftmost_longest_batch(t, **fold))
            if not self.fold:
                assert A.exists_batch(t).device == t.device and A.select_batch(t[:, :L].contiguous())[1].device == t.device
        rows_full = self.full(rows)
        assert got == rows_full
        assert ll == emul_leftmost.greedy(rows_full, self.key_len) if not self.fold else len(ll) <= len(got)
        if self.fold:
            return
        # leftmost-longest, leftmost-first, replacement, whole words
        assert triples(A.find_leftmost_longest_batch(objs, **kw)) == emul_leftmost.greedy(full, self.key_len)
        assert triples(A.find_leftmost_first_batch(objs, **kw)) == \
            first_cases.find(self.case, [list(k) for k in self.keys], hays)
        reps = [list(k[::-1]) if i % 2 else [] for i, k in enumerate(self.keys)]
        R = A.replacer({_obj(L, k): _obj(L, r) for k, r in zip(self.keys, reps)}, **kw)
        chosen = emul_leftmost.greedy(full, self.key_len)
        want_rep = [emul_replace.definition(h, [(e, k) for hh, e, k in chosen if hh == i], self.key_len, reps)
                    for i, h in enumerate(hays)]
        assert [_letters(o) for o in R.replace_batch(objs)] == want_rep
        if L == 1:
            is_word = (lambda c: c < 128 and (chr(c).isalnum() or c == 0x5F))
        else:
            is_word = (lambda c: chr(c).isalnum() or c == 0x5F)
        assert triples(A.find_all_batch(objs, whole_words=True, **kw)) == \
            emul_words.definition(hays, full, self.key_len, is_word)
        # lookups and selects against the per-key methods
        probe = [_obj(L, k) for k in self.keys[:20]] + [_obj(L, k[:-1]) for k in self.keys[:10]] + [_obj(L, [0x20])]
        assert A.exists_batch(probe, **kw).tolist() == [A.exists(k) for k in probe]
        assert A.get_batch(probe, -1, **kw) == [A.get(k, -1) for k in probe]
        assert A.longest_prefix_batch(probe, **kw).tolist() == [A.longest_prefix(k) for k in probe]
        pats = [_obj(L, k[:2]) for k in self.keys[:8]]
        assert A.keys_batch(pats, **kw) == [list(A.keys(p)) for p in pats]
        # a few stream-batch feeds: each stream reports what one scan of its whole text reports
        streams = self.text(4, 200)
        S = A.stream_batch(4, **kw)
        got = []
        cuts = [sorted(self.rng.integers(0, len(t) + 1, size=2).tolist()) for t in streams]
        for j in range(3):
            chunks = [_obj(L, t[([0] + c)[j]:(c + [len(t)])[j]]) for t, c in zip(streams, cuts)]
            got += triples(S.feed(chunks))
        assert sorted(got) == sorted(self.full(streams))
        # an iter_long().set() chain, each chunk from the root (reset)
        it = A.iter_long(_obj(L, streams[0]))
        got = [list(it)]
        for t in streams[1:]:
            it.set(_obj(L, t), True)
            got.append(list(it))
        assert got == [self.O.iter_long(_obj(L, t)) for t in streams]


PARALLEL_CELLS = [kernel_cells.Cell(1, 4, 1, 13, True), kernel_cells.Cell(1, 4, 1, 19, True),     # pair, two level-1 sizes
                  kernel_cells.Cell(1, 3, 1), kernel_cells.Cell(1, 8, 2),                           # narrow, wide placement
                  kernel_cells.Cell(4, 4, 4)]                                                       # 4-byte unicode letters
FOLD_WORDS = [b"Hello", b"HELLO", b"world", b"WoRlD", b"he", b"abc", b"ABCd", b"xyz", b"Xy"]


def _cell_job(cell, mp, seed):
    keys = kernel_cells._keys(cell, np.random.default_rng(seed))
    A = kernel_cells._build(cell, keys, mp)
    kernel_cells._check_shape(A, cell)
    return Job(A, keys, cell.L, seed)


def _fold_job(seed):
    A = pkg.flavour("bytes").Automaton(pkg.STORE_INTS)
    for i, w in enumerate(FOLD_WORDS):
        A.add_word(w, i)
    A.make_automaton()
    return Job(A, [tuple(w) for w in FOLD_WORDS], 1, seed, fold=True)


@pytest.mark.gpu
def test_independent_automata_in_parallel(monkeypatch):
    """Six threads, each with its own automaton on a different kernel or table size (the pair kernel at two level-1
    sizes, a narrow and a wide single placement, 4-byte letters, a folded table), run one mixed sequence at once:
    host lists and arrays, a 48 MiB batch on the pipelined host route, a CUDA tensor on the thread's own stream,
    leftmost-longest and -first, replacement, whole words, case folding, lookups, selects, stream feeds and an
    iter_long().set() chain.  Every result equals the reference."""
    jobs = [_cell_job(c, monkeypatch, 100 + i) for i, c in enumerate(PARALLEL_CELLS)] + [_fold_job(7)]
    _run_threads([j.run for j in jobs])


@pytest.mark.gpu
def test_one_automaton_searched_while_its_key_set_changes():
    """Several threads search one automaton while another adds a key, builds, removes it and builds again.  Every
    result is the reference of the key set before or after some change, values included; the only errors are the
    unbuilt automaton's AttributeError and a stale iterator's ValueError, as the reference raises them."""
    import torch
    base = [b"he", b"she", b"his", b"hers", b"zz", b"zzz", b"ers"]
    extra = b"rszz"
    A = pkg.flavour("bytes").Automaton()
    for k in base:
        A.add_word(k, k)
    A.make_automaton()
    hays = [b"ushers zzz his", b"hersrszzz", b"", b"rszz she zz"] * 8
    width = max(map(len, hays))
    t = torch.from_numpy(np.array([list(h.ljust(width)) for h in hays], dtype=np.uint8)).cuda()
    pad = [h.ljust(width) for h in hays]

    def answers(keys):
        O = Job._oracle(keys)
        kl = np.array([len(k) for k in keys])
        full = [(h, e, k) for h, x in enumerate(hays) for e, k in O.find_all(x)]
        padded = [(h, e, keys[k]) for h, x in enumerate(pad) for e, k in O.find_all(x)]
        first = first_cases.find("bytes", [list(k) for k in keys], [list(h) for h in hays])
        return {"find_all": [(h, e, keys[k]) for h, e, k in full], "cuda": padded,
                "leftmost_longest": [(h, e, keys[k]) for h, e, k in emul_leftmost.greedy(full, kl)],
                "leftmost_first": [(h, e, keys[k]) for h, e, k in first],
                "get": [k if k in keys else None for k in base + [extra]],
                "iter": [(e, keys[k]) for e, k in O.find_all(hays[1])]}

    allowed = [answers(base), answers(base + [extra])]
    ok_errors = (AttributeError, ValueError)

    def search():
        out = []
        calls = [("find_all", lambda: list(A.find_all_batch(hays))),
                 ("cuda", lambda: list(A.find_all_batch(t))),
                 ("leftmost_longest", lambda: list(A.find_leftmost_longest_batch(hays))),
                 ("leftmost_first", lambda: list(A.find_leftmost_first_batch(hays))),
                 ("get", lambda: A.get_batch(base + [extra], None)),
                 ("iter", lambda: list(A.iter(hays[1])))]
        for name, call in calls:
            try:
                got = call()
            except ok_errors as e:
                assert isinstance(e, AttributeError) and "Not an Aho-Corasick automaton yet" in str(e) or \
                    isinstance(e, ValueError) and "iterator is not valid anymore" in str(e), repr(e)
                continue
            if name in ("find_all", "cuda", "leftmost_longest", "leftmost_first"):
                got = [(h, e, v) for h, e, v in got]
            assert any(got == w[name] for w in allowed), (name, got[:5])
            out.append(name)
        return out

    def mutate():
        A.add_word(extra, extra)
        A.make_automaton()
        A.remove_word(extra)
        A.make_automaton()

    _run_threads([search, search, search, search, mutate])


def _cold_opt_in_child(q):
    """A fresh process: four pair-kernel automata at four level-1 sizes (one launch_pair opt-in cache, four dynamic
    shared-memory sizes) make their first scan at once from four threads, then scan once more."""
    try:
        sys.path[:0] = [ROOT, HERE]
        import kernel_cells as kc
        cells = [kc.Cell(1, 4, 1, log1, True) for log1 in kc.PAIR_LOG1]
        jobs = []
        for i, cell in enumerate(cells):
            keys = kc._keys(cell, np.random.default_rng(300 + i))

            mp = pytest.MonkeyPatch()                            # ACB_FILTER around make_automaton
            try:
                A = kc._build(cell, keys, mp)
            finally:
                mp.undo()
            kc._check_shape(A, cell)
            O = kc._oracle(cell, keys)
            text, _ = kc._text(cell, keys, np.random.default_rng(i), 1 << 20)
            off = np.array([0, len(text)], dtype=np.int64)
            jobs.append((A, text.astype(np.uint8), off, kc._want(O, cell, text, off)))
        barrier = threading.Barrier(len(jobs))
        res = [None] * len(jobs)

        def scan(i):
            A, flat, off, want = jobs[i]
            try:
                barrier.wait(timeout=120)
                first = triples(A.find_all_batch((flat, off), algo="filter"))
                again = triples(A.find_all_batch((flat, off), algo="filter"))
                res[i] = (first == want and again == want, len(want))
            except Exception:
                res[i] = (False, traceback.format_exc())
        ts = [threading.Thread(target=scan, args=(i,)) for i in range(len(jobs))]
        for th in ts:
            th.start()
        for th in ts:
            th.join(JOIN_S)
        q.put(res)
    except Exception:
        q.put([(False, traceback.format_exc())])


@pytest.mark.gpu
def test_first_shared_memory_opt_in_from_several_threads():
    """The first scans of four pair-kernel automata at four level-1 sizes, started together in a fresh process, and one
    more each: all equal the oracle.  A guard for the opt-in lock: one run cannot force the interleaving that would
    leave the cache ahead of the attribute, so the fix is argued from the code."""
    ctx = multiprocessing.get_context("spawn")
    q = ctx.Queue()
    p = ctx.Process(target=_cold_opt_in_child, args=(q,))
    p.start()
    try:
        res = q.get(timeout=JOIN_S)
        p.join(JOIN_S)
    finally:
        if p.is_alive():
            p.terminate()
            p.join(30)
    assert all(ok for ok, _ in res), res


def _gather(pool_lists, idx):
    """the concatenation of pool_lists[i] for i in idx, as an int64 array, without a Python loop over idx"""
    lens = np.array([len(x) for x in pool_lists], dtype=np.int64)
    flat = np.array([v for x in pool_lists for v in x], dtype=np.int64)
    starts = np.concatenate([[0], np.cumsum(lens)[:-1]])
    n = lens[idx]
    pos = np.repeat(starts[idx] - (np.cumsum(n) - n), n) + np.arange(int(n.sum()))
    return flat[pos]


def _lookup_case(n_rows):
    """an automaton, a pool of distinct key rows (fixed stride) and a CUDA batch of n_rows drawn from it"""
    import torch
    A = pkg.flavour("bytes").Automaton()
    keys = [b"alpha", b"alp", b"beta", b"be", b"gamma", b"delta", b"deltas"]
    for k in keys:
        A.add_word(k, k)
    A.make_automaton()
    pool = [k.ljust(8, b"\0") if i % 3 else k[:8].ljust(8, b"x") for i, k in enumerate(keys * 3)] + [b"a" * 8, b"\0" * 8]
    pool = [k[:8] for k in pool]
    rng = np.random.default_rng(5)
    idx = rng.integers(0, len(pool), size=n_rows)
    rows = np.frombuffer(b"".join(pool), dtype=np.uint8).reshape(len(pool), 8)[idx]
    return A, keys, pool, idx, torch.from_numpy(np.ascontiguousarray(rows)).cuda()


MUTATIONS = ("remove_and_build", "clear", "collect")
UNSYNCED = ("exists", "longest_prefix", "get", "select", "replace")


@pytest.mark.gpu
@pytest.mark.parametrize("mutation", MUTATIONS)
@pytest.mark.parametrize("call", UNSYNCED)
def test_unsynchronised_outputs_outlive_their_table(call, mutation):
    """A call whose CUDA output is not synchronised when it returns, made on a side stream over 64 MiB so that its kernel
    is still running; then at once remove_word + make_automaton, clear() or del + gc.collect().  After a synchronise the
    output is the answer for the key set at call time."""
    import torch
    A, keys, pool, idx, t = _lookup_case(4 << 20)                # 32 MiB of 8-byte keys
    want_pool = {"exists": [A.exists(k) for k in pool], "longest_prefix": [A.longest_prefix(k) for k in pool],
                 "get": [A.get(k, None) for k in pool], "select": [list(A.keys(k[:2])) for k in pool]}
    R = A.replacer({k: k.upper() for k in keys}) if call == "replace" else None
    if call == "select":
        t = t[:, :2].contiguous()                                # 2-letter prefixes as patterns
    if call == "replace":
        O = Job._oracle(keys)
        kl = np.array([len(k) for k in keys])
        want_pool["replace"] = [bytes(emul_replace.definition(
            list(k), [(e, kk) for _, e, kk in emul_leftmost.greedy([(0, e, kk) for e, kk in O.find_all(k)], kl)], kl,
            [list(x.upper()) for x in keys])) for k in pool]
    side = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        if call == "exists":
            out = A.exists_batch(t)
        elif call == "longest_prefix":
            out = A.longest_prefix_batch(t)
        elif call == "get":
            out = A.get_batch(t, None)
        elif call == "select":
            out = A.select_batch(t)
        else:
            out = R.replace_batch(t)
        key_objs = list(A._key_objs)
        if mutation == "remove_and_build":
            A.remove_word(b"alpha")
            A.make_automaton()
        elif mutation == "clear":
            A.clear()
        else:
            del A, R
            gc.collect()
    side.synchronize()
    if call in ("exists", "longest_prefix"):
        assert np.array_equal(out.cpu().numpy(), np.array(want_pool[call])[idx])
    elif call == "get":
        assert out == np.array(want_pool["get"], dtype=object)[idx].tolist()
    elif call == "select":
        offs, ids = (x.cpu().numpy() for x in out)
        kid = {k: i for i, k in enumerate(key_objs)}
        pool_ids = [[kid[k] for k in w] for w in want_pool["select"]]
        assert np.array_equal(np.diff(offs), np.array([len(w) for w in pool_ids])[idx])
        assert np.array_equal(ids, _gather(pool_ids, idx))
    else:
        flat, offs = (x.cpu().numpy() for x in out)
        assert flat.tobytes() == b"".join(np.array(want_pool["replace"], dtype=object)[idx].tolist())


# ====================================================================== C. two devices
def _entry_points(dev):
    """(name, call) for every kind of entry point, each naming device `dev` (or a tensor on it)"""
    import torch
    hays = [b"ushers his", b"hershe", b"", b"she sells"]
    rng = np.random.default_rng(3)
    big = rng.choice(np.frombuffer(b"#%&*+-hes", dtype=np.uint8), size=40 * MiB)           # the pipelined host route
    big_off = np.array([0, 3 * MiB, 32 * MiB, 40 * MiB], dtype=np.int64)

    def make():
        A = pkg.flavour("bytes").Automaton()
        for k in (b"he", b"she", b"his", b"hers"):
            A.add_word(k, k)
        A.make_automaton()
        return A
    A = make()
    t = torch.from_numpy(np.frombuffer(b"ushers his hershe", dtype=np.uint8).reshape(1, -1).copy()).to(f"cuda:{dev}")

    def streams():
        S = A.stream_batch(2, device=dev)
        S.feed(hays[:2])
        S.positions
        S.reset()
        T = A.stream_batch(2, device=dev, leftmost_longest=True)
        T.feed(hays[:2])
        T.finish()
        del S, T
        gc.collect()

    def first_tensor():
        B = make()
        B.find_all_batch(t)                                      # the upload
        B.find_all_batch(t)

    def key_change():
        A.add_word(b"zz", b"zz")
        A.make_automaton()
        A.find_all_batch(hays, device=dev)

    def collect():
        B = make()
        B.find_all_batch(hays, device=dev)
        del B
        gc.collect()

    return [("find_all", lambda: A.find_all_batch(hays, device=dev)),
            ("pipelined", lambda: A.find_all_batch((big, big_off), device=dev)),
            ("leftmost", lambda: (A.find_leftmost_longest_batch(hays, device=dev), A.find_leftmost_first_batch(hays, device=dev))),
            ("lookups", lambda: (A.exists_batch(hays, device=dev), A.get_batch(hays, None, device=dev),
                                 A.longest_prefix_batch(hays, device=dev))),
            ("select", lambda: A.select_batch([b"h", b"s"], device=dev)),
            ("replacer", lambda: A.replacer(device=dev).replace_batch(hays)),
            ("streams", streams),
            ("tensor_first", first_tensor),
            ("tensor", lambda: (A.find_all_batch(t), A.find_leftmost_longest_batch(t), A.exists_batch(t))),
            ("key_change", key_change),
            ("collect", collect)]


@pytest.mark.gpu
@two_gpus
def test_current_device_is_preserved():
    """Every entry point, run with device=1 while the current device is 0 and, from a thread whose current device is 1,
    with device=0, leaves the current device as it was."""
    import torch

    def check(home, dev):
        torch.cuda.set_device(home)
        moved = []
        for name, call in _entry_points(dev):
            call()
            torch.cuda.synchronize(dev)
            if torch.cuda.current_device() != home:
                moved.append(name)
                torch.cuda.set_device(home)
        return moved

    torch.cuda.set_device(0)
    try:
        assert check(0, 1) == []
        assert _run_threads([lambda: check(1, 0)]) == [[]]
    finally:
        torch.cuda.set_device(0)


@pytest.mark.gpu
@two_gpus
def test_every_feature_on_device_one(monkeypatch):
    """The mixed sequence of the thread test on device 1 while the current device is 0, tensors on cuda:1 included"""
    import torch
    torch.cuda.set_device(0)
    for job in [_cell_job(PARALLEL_CELLS[0], monkeypatch, 11), _cell_job(PARALLEL_CELLS[4], monkeypatch, 12), _fold_job(13)]:
        job.run(device=1)
        assert torch.cuda.current_device() == 0


@pytest.mark.gpu
@two_gpus
def test_one_automaton_moves_between_devices():
    """One automaton alternates between the devices (its table is uploaded again on each switch): a stream batch on
    device 0 fed between calls on device 1 reports what the oracle reports for each whole stream, and one Replacer gives
    the same output on both devices."""
    import torch
    keys = [b"he", b"she", b"his", b"hers", b"shell"]
    A = pkg.flavour("bytes").Automaton(pkg.STORE_INTS)
    for i, k in enumerate(keys):
        A.add_word(k, i)
    A.make_automaton()
    O = Job._oracle(keys)
    hays = [b"ushers", b"his shell", b"sheshe"]
    S = A.stream_batch(2, device=0)
    texts = [b"she sells sea shells", b"hishershe"]
    got = []
    for j in range(3):
        chunks = [t[j * 7:(j + 1) * 7] for t in texts]
        got += triples(S.feed(chunks))
        w = [(h, e, k) for h, x in enumerate(hays) for e, k in O.find_all(x)]
        assert triples(A.find_all_batch(hays, device=1)) == w
    assert sorted(got) == sorted((h, e, k) for h, x in enumerate(texts) for e, k in O.find_all(x))
    R = A.replacer({k: k.upper() for k in keys}, device=0)
    host = R.replace_batch(hays)
    rows = np.array([list(h.ljust(9)) for h in hays], dtype=np.uint8)
    flat, offs = R.replace_batch(torch.from_numpy(rows).to("cuda:1"))
    assert flat.device.index == 1
    out = flat.cpu().numpy().tobytes()
    o = offs.cpu().numpy().tolist()
    assert [out[o[i]:o[i + 1]].rstrip(b" ") for i in range(len(hays))] == host


@pytest.mark.gpu
@two_gpus
def test_a_thread_per_device(monkeypatch):
    """One thread per device, each with its own automaton, at once"""
    jobs = [_cell_job(PARALLEL_CELLS[1], monkeypatch, 21), _cell_job(PARALLEL_CELLS[3], monkeypatch, 22)]
    _run_threads([lambda: jobs[0].run(device=0), lambda: jobs[1].run(device=1)])


def _nccl_rank(rank, port, q):
    try:
        sys.path[:0] = [ROOT, HERE]
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE="2")
        import torch
        import torch.distributed as dist
        from pyahocorasick_b200 import distributed as D
        from pyahocorasick_b200 import synth
        torch.cuda.set_device(rank)
        dist.init_process_group("nccl", rank=rank, world_size=2)
        try:
            rng = np.random.Generator(np.random.PCG64(77))
            keys = synth.draw_keys(rng, synth.ALNUM, 300, 4, 9)
            n_hay = 1001
            hay = synth.random_haystacks(rng, synth.ALNUM, n_hay, 64)
            synth.plant(rng, hay, keys, np.arange(n_hay))
            A = synth.build_automaton(keys)
            O = Job._oracle(keys)
            want = O.scan_batch_bytes(hay.reshape(-1), np.arange(n_hay + 1, dtype=np.int64) * 64).astype(np.int64)
            lo, hi = D.shard_bounds(n_hay, 2, rank)
            sm = D.scan_sharded(A, hay)
            ok = np.array_equal(D.gather_records(sm), want) and sm.total == len(want)
            loc = D.scan_sharded(A, hay[lo:hi], already_local=True, n_global=n_hay)
            ok = ok and np.array_equal(D.gather_records(loc), want)
            mine = want[(want[:, 0] >= lo) & (want[:, 0] < hi)]
            ok = ok and np.array_equal(np.stack([loc.hay_id, loc.end_index, loc.key_id], axis=1).astype(np.int64), mine)
            q.put((rank, bool(ok), len(want)))
        finally:
            dist.destroy_process_group()
    except Exception:
        q.put((rank, False, traceback.format_exc()))


@pytest.mark.gpu
@two_gpus
def test_scan_sharded_over_nccl():
    """scan_sharded + gather_records on two ranks, one device each, with the real kernels: the global and the
    already_local forms give the oracle's full list"""
    ctx = multiprocessing.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + os.getpid() % 2000
    procs = [ctx.Process(target=_nccl_rank, args=(r, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    try:
        res = [q.get(timeout=JOIN_S) for _ in procs]
        for p in procs:
            p.join(JOIN_S)
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
                p.join(30)
    assert all(r[1] for r in res), res
