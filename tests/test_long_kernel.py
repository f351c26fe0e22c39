"""acb_long_kernel (ACB_ALGO_LONG: iter_long / find_long_batch) against the C oracle, record for record.

The kernel replays the reference's longest-match state machine (src/AutomatonSearchIterLong.c:89-153) once per
haystack: trie edges letter by letter, letter-level fail links, and the early return when a non-terminal state's fail
state ends a key.  The cells cross letter widths with key sets that reach each branch of that machine:

  widths    1-byte letters (bytes), 2-byte letters (bytes flavour KEY_SEQUENCE), 4-byte letters (unicode str, and
            unicode KEY_SEQUENCE with values above 0xFFFF).  The letters of the wider alphabets share their low (first,
            little-endian) bytes, so the byte-level fail chain of a letter-aligned state passes through states inside a
            letter, which the letter-level walk must skip (letter_fail).
  key sets  keys that are prefixes of longer keys (a match is pending when a mismatch comes); non-terminal states whose
            fail state ends a key (the early return); fail chains several states deep without a key on them; random.

  GPU (-m gpu)  ragged batches of 700 haystacks (more than one 256-thread block, not a multiple of it) with empty
                haystacks first, in runs and last, haystacks that are exactly one key, matches at the first and the last
                letter; fixed strides of a power of two and not; the list entry point; sort=False as a multiset; one
                haystack of 3 MiB.  Plus an iter_long() stream whose chunk overflows the record buffer after it was
                entered in a non-root state, and the C ABI's one-shot start state (acb_table_set_long_state /
                acb_table_get_long_state) over a multi-haystack batch and over empty scans.
  CPU           the same tables through tests/emul.py's emul_long, so that a failing GPU cell shows whether the tables
                or the kernel are wrong.
"""
import ctypes

import numpy as np
import pytest

import emul
import oracle
import pyahocorasick_b200 as ac
from batch_cases import DT, triples
from pyahocorasick_b200 import _native as N

# name -> (letter bytes, flavour, KEY_SEQUENCE, alphabet a b c d, a letter in no key)
WIDTHS = {
    "L1": (1, "bytes", False, (0x42, 0x61, 0xE9, 0x00), 0x7A),
    "L2": (2, "bytes", True, (0x0042, 0x4242, 0x4200, 0x0061), 0x7A7A),
    "L4": (4, "unicode", False, (0x42, 0x142, 0x4242, 0x1F642), 0x7A),
    "L4seq": (4, "unicode", True, (0x42, 0x10042, 0x4242, 0xFFFF0042), 0x7A7A7A7A),
}

# key sets over the alphabet's indices
KEYSETS = {
    "prefixes": [(0,), (0, 1), (0, 1, 0, 1), (0, 1, 0, 1, 2), (1, 2), (1, 2, 3, 3), (2,), (2, 2, 2, 2, 2), (3, 0, 3, 0, 3, 0)],
    # (0,3) fails to the key (3,); (2,0,2) fails to the key (0,2); (0,1,2) fails to the key (1,2)
    "fail_ends_key": [(0, 1, 2, 3), (1, 2), (0, 3, 1, 1), (3,), (2, 0, 2, 0, 1), (0, 2)],
    "deep_fail": [(0, 1, 0, 1, 0, 1, 2), (0, 0, 0, 0, 0, 3), (1, 0, 1, 0, 1, 3), (0, 1, 2, 0, 1, 2, 0, 1, 3), (3, 3)],
    "random": None,
}


def _keys(width, keyset, rng):
    alpha = WIDTHS[width][3]
    ks = KEYSETS[keyset]
    if ks is None:
        ks = [tuple(int(x) for x in rng.integers(0, 4, size=int(rng.integers(1, 8)))) for _ in range(30)]
    return list(dict.fromkeys(tuple(alpha[i] for i in k) for k in ks))


def _pkg_key(width, k):
    L, fl, seq = WIDTHS[width][:3]
    if seq:
        return tuple(k)
    return bytes(k) if L == 1 else "".join(map(chr, k))


def _build(width, keys):
    L, fl, seq = WIDTHS[width][:3]
    mod = ac.flavour(fl)
    A = mod.Automaton(mod.STORE_INTS, mod.KEY_SEQUENCE) if seq else mod.Automaton(mod.STORE_INTS)
    for i, k in enumerate(keys):
        A.add_word(_pkg_key(width, k), i)
    A.make_automaton()
    assert A.flat()["letter_bytes"] == L
    return A


def _oracle(keys):
    O = oracle.OracleAutomaton()
    for i, k in enumerate(keys):
        O.add_word(tuple(k), i)
    O.make_automaton()
    return O


def _text(width, keys, rng, n):
    """n letters: mostly the alphabet, some letters of no key, keys planted back to back in places"""
    alpha, foreign = WIDTHS[width][3], WIDTHS[width][4]
    t = np.asarray(alpha, dtype=np.uint32)[rng.integers(0, 4, size=n)]
    t[rng.random(n) < 0.05] = foreign
    i = 0
    while i < n:
        i += int(rng.integers(0, 24))
        k = keys[int(rng.integers(0, len(keys)))]
        if i + len(k) <= n:
            t[i:i + len(k)] = k
        i += len(k)
    return t


def _ragged(width, keys, rng, n_hay):
    """letters and offsets (in letters) of n_hay haystacks: empty ones first, in runs and last, some exactly one key,
    keys at the first and at the last letter of others"""
    lens = rng.integers(0, 60, size=n_hay)
    for a, b in ((0, 3), (50, 55), (n_hay // 2, n_hay // 2 + 3), (n_hay - 2, n_hay)):
        lens[a:b] = 0
    whole = {h: keys[j % len(keys)] for j, h in enumerate(range(7, n_hay - 2, 23))}    # haystacks that are one key
    for h, k in whole.items():
        lens[h] = len(k)
    off = np.zeros(n_hay + 1, dtype=np.int64)
    np.cumsum(lens, out=off[1:])
    t = _text(width, keys, rng, int(off[-1]))
    for h in range(n_hay):
        a, b = int(off[h]), int(off[h + 1])
        k = whole.get(h, keys[(h * 7) % len(keys)])
        if h in whole:
            t[a:b] = k
        elif h % 5 == 0 and b - a >= len(k):                # a key at the first letter
            t[a:a + len(k)] = k
        elif h % 5 == 1 and b - a >= len(k):                # ... at the last letter
            t[b - len(k):b] = k
    return t, off


def _flat(width, letters):
    return np.ascontiguousarray(letters.astype(DT[WIDTHS[width][0]])).view(np.uint8)


def _diff(got, want):
    i = next((i for i, (a, b) in enumerate(zip(got, want)) if a != b), min(len(got), len(want)))
    sg, sw = set(got), set(want)
    return (f"{len(got)} records, want {len(want)}; first difference at {i}: got {got[i:i + 3]}, want {want[i:i + 3]}; "
            f"missing {sorted(sw - sg)[:5]}, extra {sorted(sg - sw)[:5]}")


def _check(got, want, what):
    if got != want:
        pytest.fail(f"{what}: {_diff(got, want)}")


def _hay_objects(width, letters, off):
    """the list entry point's haystacks: bytes, tuples or str"""
    L, fl, seq = WIDTHS[width][:3]
    out = []
    for h in range(len(off) - 1):
        seg = letters[int(off[h]):int(off[h + 1])]
        if seq:
            out.append(tuple(int(x) for x in seg))
        elif L == 1:
            out.append(seg.astype(np.uint8).tobytes())
        else:
            out.append("".join(map(chr, seg.tolist())))
    return out


CELLS = [(w, k) for w in WIDTHS for k in KEYSETS]
IDS = [f"{w}-{k}" for w, k in CELLS]


def _seed(width, keyset):
    return sum(f"{width}/{keyset}".encode()) * 7919


# ------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize("width, keyset", CELLS, ids=IDS)
def test_long_kernel_matches_oracle(width, keyset):
    rng = np.random.Generator(np.random.PCG64(_seed(width, keyset)))
    keys = _keys(width, keyset, rng)
    A, O = _build(width, keys), _oracle(keys)
    L = WIDTHS[width][0]
    # ragged, 700 haystacks: three 256-lane blocks, the last one partly idle
    t, off = _ragged(width, keys, rng, 700)
    want = O.iter_long_batch_letters(t, off)
    assert len(want) > 700
    assert any(e == len(keys[v]) - 1 for _, e, v in want)                         # a match at the first letter
    assert any(e == off[h + 1] - off[h] - 1 for h, e, _ in want)                 # ... and at the last
    assert any(e == len(keys[v]) - 1 == off[h + 1] - off[h] - 1 for h, e, v in want)   # a key as long as its haystack
    batch = (_flat(width, t), off * L)
    _check(triples(A.find_long_batch(batch)), want, "ragged")
    _check(sorted(triples(A.find_long_batch(batch, sort=False))), sorted(want), "ragged, unsorted")
    # the list entry point
    hays = _hay_objects(width, t, off[:301])
    _check(triples(A.find_long_batch(hays)), [r for r in want if r[0] < 300], "list")
    # fixed strides: a power of two and not
    for stride in (64, 37):
        n_hay = 300
        ft = _text(width, keys, rng, stride * n_hay)
        foff = np.arange(n_hay + 1, dtype=np.int64) * stride
        fw = O.iter_long_batch_letters(ft, foff)
        rows = _flat(width, ft).reshape(n_hay, stride * L)
        _check(triples(A.find_long_batch(rows)), fw, f"stride {stride}")


@pytest.mark.gpu
@pytest.mark.parametrize("width", list(WIDTHS))
def test_long_kernel_long_haystack(width):
    """one haystack of 3 MiB between two short ones: one lane walks it all"""
    rng = np.random.Generator(np.random.PCG64(_seed(width, "long")))
    keys = _keys(width, "random", rng)
    A, O = _build(width, keys), _oracle(keys)
    L = WIDTHS[width][0]
    n = (3 << 20) // L
    t = _text(width, keys, rng, n + 200)
    off = np.array([0, 100, 100 + n, n + 200], dtype=np.int64)
    want = O.iter_long_batch_letters(t, off)
    _check(triples(A.find_long_batch((_flat(width, t), off * L))), want, "3 MiB haystack")


def _stream(A):
    """iter_long() over three chunks: the second is entered in the state "ab" and holds over 4096 matches"""
    it = A.iter_long(b"zzab")
    out = list(it)
    it.set(b"cd" + b"q" * 5000 + b"ab")
    out += list(it)
    it.set(b"cdq")
    return out + list(it)


def _stream_automaton():
    A = ac.flavour("bytes").Automaton(ac.STORE_INTS)
    for i, k in enumerate([b"abcd", b"q", b"cd"]):
        A.add_word(k, i)
    A.make_automaton()
    return A


@pytest.mark.gpu
def test_iter_long_stream_overflow_retry_keeps_the_start_state(monkeypatch):
    """the record buffer of a fresh automaton holds 4096 records: the second chunk overflows it, and the retry must
    start in the carried state again ("abcd" straddles the seam) -- equal to a run with a large buffer and to the
    emulated kernel"""
    fresh = _stream_automaton()
    got = _stream(fresh)
    assert fresh._match_cap > 5000                     # the retry happened
    big = _stream_automaton()
    big._match_cap = 1 << 16
    assert got == _stream(big)
    with monkeypatch.context() as m:
        emul.install(m, "filter")
        want = _stream(_stream_automaton())
    assert got == want
    assert got[:2] == [(4 + 1, 0), (4 + 2, 1)] and len(got) == 5003


def _state(f, text):
    """the trie state reached from the root over `text` (1-byte letters)"""
    s = 0
    for b in text:
        s = int(f["goto_cm"][f["byte_class"][b], s])
        assert s >= 0
    return s


@pytest.mark.gpu
def test_c_abi_one_shot_long_state():
    """acb_table_set_long_state applies to haystack 0 of the next ACB_ALGO_LONG scan only; every other haystack and the
    scan after it start at the root; acb_table_get_long_state is the state haystack 0 ended in.  Through
    acb_scan_host and acb_scan_device, against emul_long with the same start state.  An empty scan consumes the state:
    haystack 0 ends where it started."""
    import torch
    A = _stream_automaton()
    f = A.flat()
    tb = A._ensure_table(0)
    lib = N.lib()
    s = _state(f, b"ab")
    found = ctypes.c_int64(0)
    st = ctypes.c_int32(-1)

    def get_state():
        N.check(lib.acb_table_get_long_state(tb, ctypes.byref(st)))
        return st.value

    def host_scan(flat, off):
        out = np.full((64 + 16, 3), -1, dtype=np.int32)
        N.check(lib.acb_scan_host(tb, N.ptr(flat) if flat.size else None, flat.size, N.ptr(off), len(off) - 1, 0,
                                  N.ptr(out), 64, ctypes.byref(found), N.ALGO_LONG, 1))
        assert (out[found.value:] == -1).all()
        return [tuple(r) for r in out[:found.value].tolist()], get_state()

    def device_scan(flat, off):
        d_hay = torch.from_numpy(flat.copy() if flat.size else np.zeros(16, np.uint8)).cuda()
        d_off = torch.from_numpy(off).cuda()
        d_out = torch.full((64 + 16, 3), -1, dtype=torch.int32, device="cuda")
        d_cnt = torch.zeros(1, dtype=torch.int64, device="cuda")
        stream = torch.cuda.current_stream()
        N.check(lib.acb_scan_device(tb, d_hay.data_ptr(), flat.size, d_off.data_ptr(), len(off) - 1, 0, d_out.data_ptr(),
                                    64, d_cnt.data_ptr(), stream.cuda_stream, N.ALGO_LONG))
        stream.synchronize()
        n = int(d_cnt.item())
        out = d_out.cpu().numpy()
        assert (out[n:] == -1).all()
        rec = out[:n]
        rec = rec[np.lexsort((rec[:, 1], rec[:, 0]))]
        return [tuple(r) for r in rec.tolist()], get_state()

    batches = [[b"c", b"cdab", b"", b"abcdcd"],                 # haystack 0 ends in "abc" from s, in "c" from the root
               [b"cdxq", b"cdab", b"q"],                        # haystack 0 completes "abcd" from s, "cd" from the root
               [b"", b"cdab"]]                                  # haystack 0 empty: ends where it started
    for hays in batches:
        flat = np.frombuffer(b"".join(hays), dtype=np.uint8)
        off = np.concatenate([[0], np.cumsum([len(h) for h in hays])]).astype(np.int64)
        from_s = emul.emul_long(f, flat, off, 0, init_state=s, want_state=True)
        from_root = emul.emul_long(f, flat, off, 0, init_state=0, want_state=True)
        assert from_s != from_root
        for scan in (host_scan, device_scan):
            N.check(lib.acb_table_set_long_state(tb, s))
            assert scan(flat, off) == from_s, (hays, scan.__name__)
            assert scan(flat, off) == from_root, (hays, scan.__name__)        # the state was one shot
    # an empty scan consumes the state and reports it as the end state of haystack 0
    hays = [b"cdab", b"cd"]
    flat = np.frombuffer(b"".join(hays), dtype=np.uint8)
    off = np.array([0, 4, 6], dtype=np.int64)
    from_root = emul.emul_long(f, flat, off, 0, init_state=0, want_state=True)
    empty = np.empty(0, dtype=np.uint8)
    for scan in (host_scan, device_scan):
        for eoff in (np.array([0, 0, 0], dtype=np.int64), np.array([0], dtype=np.int64)):      # empty haystacks, none
            N.check(lib.acb_table_set_long_state(tb, s))
            assert scan(empty, eoff) == ([], s), (scan.__name__, eoff)
            assert scan(flat, off) == from_root, (scan.__name__, eoff)


# ------------------------------------------------------------------ CPU: the same tables through the emulation
@pytest.mark.parametrize("width, keyset", CELLS, ids=IDS)
def test_long_tables_match_oracle_emulated(width, keyset):
    rng = np.random.Generator(np.random.PCG64(_seed(width, keyset)))
    keys = _keys(width, keyset, rng)
    A, O = _build(width, keys), _oracle(keys)
    L = WIDTHS[width][0]
    t, off = _ragged(width, keys, rng, 120)
    want = O.iter_long_batch_letters(t, off)
    assert len(want) > 100
    _check(emul.emul_long(A.flat(), _flat(width, t), off * L, 0), want, "emulated ragged")
    ft = _text(width, keys, rng, 37 * 20)
    foff = np.arange(21, dtype=np.int64) * 37
    _check(emul.emul_long(A.flat(), _flat(width, ft), None, 37 * L), O.iter_long_batch_letters(ft, foff), "emulated stride")


def test_wide_letter_tables_have_fail_links_inside_letters():
    """the alphabets of the wider widths do what they are for: some letter-aligned state's byte-level fail link lands
    inside a letter, where the letter-level one must not"""
    for width in ("L2", "L4", "L4seq"):
        rng = np.random.Generator(np.random.PCG64(_seed(width, "random")))
        A = _build(width, _keys(width, "random", rng))
        f = A.flat()
        L = WIDTHS[width][0]
        depth = np.zeros(f["n_states"], dtype=np.int64)
        for s in range(f["n_states"]):                      # BFS ids: a child's id is larger than its parent's
            ch = f["goto_cm"][:, s]
            depth[ch[ch >= 0]] = depth[s] + 1
        aligned = [s for s in range(1, f["n_states"]) if depth[s] % L == 0]
        assert any(depth[f["fail"][s]] % L for s in aligned), width
        assert all(depth[f["letter_fail"][s]] % L == 0 for s in aligned), width


def test_iter_long_stream_overflow_retry_emulated(monkeypatch):
    emul.install(monkeypatch, "filter")
    got = _stream(_stream_automaton())
    assert got[:2] == [(4 + 1, 0), (4 + 2, 1)] and len(got) == 5003
