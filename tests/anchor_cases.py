"""Key sets built from the anchor hash so that the anchor table's rare chains are certain to exist, the properties
read back from a built table, and texts that send candidates into those chains; shared by test_anchor_table.py.  Not a
test module.

The anchor tag of a gram is hash2(gram) | 1 (acb_hash.h), its home slot the top logA bits.  Window 0 of a gram of at
least 4 bytes is a whole 32-bit word with an odd multiplier, so for any target tag t and any other windows there is
exactly one window 0 per h in {t, t - 1}: grams with a chosen tag (and twins: other grams with a key gram's tag) are
solved, not searched.  A gram of 1-3 bytes fills one window whose multiplier is shifted by its unused bytes: the tag is
then a bijection of the gram (no twins), and grams with a chosen home slot are picked from all grams.  Code points stop
at U+10FFFF, so a one-letter unicode gram has no twin either, and window 0 of a longer one is solved for many random
other windows until it is a code point.

What a key set holds (where the cell's gram g, stride s and letter width L allow it):
  wrap        tags homed in the last slot, with entries enough to carry the chain over slot 0
  wrap-split  one tag with entries on both sides of the wrap
  uu / um / mm  twin grams under one tag: UNIQUE + UNIQUE at one j, UNIQUE + MULTI, MULTI + MULTI
  two-j       one tag at two probe offsets j (stride > L)
  displaced   a tag whose one entry (UNIQUE, j = 0) sits behind a foreign tag's entry in its home slot
  run8        a tag behind at least 8 foreign entries from its home slot on
  shared / long / k20 / k21   MULTI entries of a shared prefix and of one key longer than 20 bytes; keys of exactly 20
              bytes (UNIQUE) and of the next whole letter past 20 (MULTI)
  one-tag     several entries of one tag without twins (one gram at several j, several UNIQUE nodes under one (j, gram))
"""
import collections
import dataclasses

import numpy as np

import emul
import kernel_cells as kc
from kernel_cells import Cell

M32 = 0xFFFFFFFF
DT = {1: np.uint8, 2: "<u2", 4: "<u4"}


@dataclasses.dataclass(frozen=True)
class ACell:
    """a kernel_cells cell; seq: 4-byte letters as a unicode KEY_SEQUENCE (any 32-bit letter) instead of str"""
    cell: Cell
    seq: bool = False

    def __getattr__(self, k):
        return getattr(self.cell, k)

    @property
    def name(self):
        return self.cell.name + ("-seq" if self.seq else "")


CELLS = [ACell(c) for c in kc.CELLS] + [ACell(Cell(4, g, s), seq=True) for g in (4, 8, 12, 16) for s in (4, 16)]
IDS = [c.name for c in CELLS]


def _letters(c):
    return c.g // c.L


def _min_letters(c):
    return (c.g + c.s - c.L) // c.L


def _max_unique(c):
    """letters of the longest key an entry can carry (20 bytes)"""
    return 20 // c.L


def has_twins(c):
    return c.g >= 4 and not (c.L == 4 and not c.seq and c.g == 4)


def capabilities(c):
    """the properties the cell's shape allows (the module docstring names them)"""
    uniq = _min_letters(c) <= _max_unique(c)
    multi_j = c.s > c.L
    caps = {"mm", "shared", "long"}
    if has_twins(c):
        caps |= {"uu", "um"} if uniq else set()
    elif multi_j:
        caps.add("one-tag")
    if multi_j:
        caps.add("two-j")
    if c.g >= 2 or multi_j:
        caps.add("wrap")
    if has_twins(c) or multi_j:
        caps.add("wrap-split")
    if c.g >= 2:
        caps.add("run8")
        if uniq:
            caps.add("displaced")
    if _min_letters(c) * c.L <= 20:
        caps.add("k20")
    if _min_letters(c) <= 20 // c.L + 1:
        caps.add("k21")
    if not has_twins(c) and not multi_j:
        caps.discard("mm")                   # one gram per tag and one j: a tag has one entry
    return caps


# ------------------------------------------------------------------ letters, grams, hashes
def valid(c, x):
    """letters of the cell's key type: bytes, 16-bit sequence items, any 32-bit item, or a code point (no surrogate)"""
    x = np.asarray(x, dtype=np.int64)
    if c.L == 1:
        return (x >= 0) & (x <= 0xFF)
    if c.L == 2:
        return (x >= 0) & (x <= 0xFFFF)
    if c.seq:
        return (x >= 0) & (x <= M32)
    return (x >= 0) & (x <= 0x10FFFF) & ((x < 0xD800) | (x > 0xDFFF))


def random_letters(c, rng, shape):
    if c.L == 1:
        return rng.integers(0, 256, size=shape, dtype=np.int64)
    if c.L == 2:
        return rng.integers(0, 1 << 16, size=shape, dtype=np.int64)
    if c.seq:
        return rng.integers(0x100, 1 << 32, size=shape, dtype=np.int64)
    x = rng.integers(0x100, 0x10F800, size=shape, dtype=np.int64)       # above latin-1, surrogates moved to the top
    return np.where(x >= 0xD800, x + 0x800, x)


def _bytes(c, letters):
    return np.asarray(letters, dtype=np.int64).astype(DT[c.L]).view(np.uint8)


def _windows(c, grams):
    """(N, gl) letters -> (N, nw) little-endian 32-bit windows (zero past the gram), as uint64"""
    grams = np.atleast_2d(np.asarray(grams, dtype=np.int64))
    b = grams.astype(DT[c.L]).view(np.uint8).reshape(len(grams), c.g)
    nw = (c.g + 3) // 4
    pad = np.zeros((len(grams), 4 * nw), dtype=np.uint8)
    pad[:, :c.g] = b
    return pad.view("<u4").astype(np.uint64)


def hash_many(c, grams, stage):
    """acb_hash_bytes_wide of every gram: the low half is hash 1 / hash 2"""
    W = _windows(c, grams)
    mul = emul.multipliers(c.g, stage)
    h = np.zeros(len(W), dtype=np.uint64)
    for k in range(W.shape[1]):
        h += W[:, k] * np.uint64(mul[k])
    return h


def tags(c, grams):
    return (hash_many(c, grams, 2) & np.uint64(M32)) | np.uint64(1)


def tag_of(c, gram):
    return int(tags(c, [gram])[0])


def _inv(x):
    return pow(int(x), -1, 1 << 32)


def solve(c, t, rng, n, avoid=()):
    """n distinct grams (letter tuples) of tag t, none in `avoid`: window 0 solved for random other windows"""
    assert has_twins(c)
    w0n = 4 // c.L                                       # letters in window 0
    mul = emul.multipliers(c.g, 2)
    inv0 = _inv(mul[0])
    out, seen = [], set(avoid)
    for _ in range(64):
        N = 64 if (c.L < 4 or c.seq) else 1 << 15
        rest = random_letters(c, rng, (N, _letters(c) - w0n))
        grams = np.concatenate([np.zeros((N, w0n), dtype=np.int64), rest], axis=1)
        h_rest = hash_many(c, grams, 2) & np.uint64(M32)
        for h in (t, t - 1):
            w0 = ((np.uint64(h) - h_rest) & np.uint64(M32)) * np.uint64(inv0) & np.uint64(M32)
            if c.L == 4:
                lets = w0[:, None].astype(np.int64)
            else:
                lets = w0[:, None].astype("<u4").view(DT[c.L]).reshape(N, w0n).astype(np.int64)
            ok = np.all(valid(c, lets), axis=1) & (lets.max(axis=1) > (0xFF if c.L == 4 else -1))
            for a, r in zip(lets[ok], rest[ok]):
                gram = tuple(int(x) for x in a) + tuple(int(x) for x in r)
                if gram not in seen:
                    seen.add(gram)
                    out.append(gram)
            if len(out) >= n:
                out = out[:n]
                assert all(tag_of(c, x) == t for x in out)
                return out
    raise AssertionError(f"{c.name}: no {n} grams of tag {t:#x}")


def _pool(c, rng):
    """grams to pick home slots from, when the tag is a bijection of the gram: all of them, or a large sample"""
    if c.L == 1 and c.g == 1:
        return np.arange(256, dtype=np.int64)[:, None]
    if c.g == 2:                                         # two bytes or one 16-bit letter: all 65 536
        x = np.arange(1 << 16, dtype=np.int64)
        return x[:, None] if c.L == 2 else np.stack([x & 0xFF, x >> 8], axis=1)
    if c.L == 4:                                         # one code point: all of them above latin-1
        x = np.arange(0x100, 0x110000, dtype=np.int64)
        return x[valid(c, x)][:, None]
    return random_letters(c, rng, (1 << 20, _letters(c)))


def bucket(c, top12, n, rng, avoid=()):
    """n grams whose tags share the top 12 bits `top12` (one home slot for logA <= 12), in increasing tag order: the
    order in which the table inserts them, so the last comes behind the others"""
    if has_twins(c):
        return [solve(c, (top12 << 20) | 0x1001 | (2 * i), rng, 1, avoid)[0] for i in range(n)]
    P = _pool(c, rng)
    T = tags(c, P)
    sel = np.nonzero((T >> np.uint64(20)) == np.uint64(top12))[0]
    sel = sel[np.argsort(T[sel], kind="stable")]
    grams = [tuple(int(x) for x in P[i]) for i in sel if tuple(int(x) for x in P[i]) not in avoid]
    assert len(grams) >= n, (c.name, top12, len(grams))
    idx = np.sort(rng.choice(len(grams), size=n, replace=False))
    return [grams[i] for i in idx]


def last_home_gram(c):
    """the 1-byte gram whose home slot is the highest (1-byte grams have homes 2^(logA-8) slots apart)"""
    P = _pool(c, None)
    return (int(P[int(np.argmax(tags(c, P)))][0]),)


# ------------------------------------------------------------------ the key set
@dataclasses.dataclass
class Plan:
    keys: list                   # letter tuples; key id = index
    roles: dict                  # property -> the letter tuples of the keys that give it
    near: list                   # key letters with the last letter changed: the gram's tag, other text
    decoys: list                 # (gram, tag): text grams that are no key gram, with a key gram's tag
    twins: dict                  # decoy gram -> the key gram with its tag


def build_plan(c, rng, lA=10):
    L, gl, m, U = c.L, _letters(c), _min_letters(c), _max_unique(c)
    sl = c.s // L
    ctx = kc.ALPHA[L] if L < 4 else [0x142, 0x1F600]

    def rnd(n):
        return tuple(int(x) for x in rng.choice(ctx, size=n))

    keys, roles, used = [], {}, set()

    def add(role, k):
        k = tuple(k)
        assert len(k) >= m, (role, k, m)
        if k not in keys:
            keys.append(k)
        roles.setdefault(role, []).append(k)
        return k

    def short(gram, j=0, n=None):
        """a key with `gram` at offset j of exactly n (default: the shortest) letters"""
        n = max(m, j + gl) if n is None else n
        return rnd(j) + tuple(gram) + rnd(n - j - gl)

    def multi(role, gram, j=0):
        """two keys through the node of (j, gram): a MULTI entry"""
        base = rnd(j) + tuple(gram)
        pad = rnd(max(0, m - len(base)))
        add(role, base + pad + (ctx[0],))
        add(role, base + pad + (ctx[1],) + rnd(1))

    def fresh():
        """a gram no key starts with yet: the node below it carries this key alone"""
        while True:
            gram = tuple(int(x) for x in random_letters(c, rng, gl))
            if gram not in used and all(k[:gl] != gram for k in keys):
                used.add(gram)
                return gram

    uniq = m <= U
    twins = {}
    # shape: the shortest key length is what forces (g, s)
    add("shape", rnd(m))
    # wrap: three tags homed in the last slot for logA <= 12, the first with entries on both sides of the wrap
    if has_twins(c):
        for i in range(3):                              # the lowest tags homed in the last slot: inserted first
            t = (((1 << lA) - 1) << (32 - lA)) | 1 | (2 * i)
            for gram in solve(c, t, rng, (2 if c.g == 4 else 4) if i == 0 else 1, used):
                used.add(gram)
                add("wrap", short(gram) if uniq else short(gram, n=m + 1))
    elif c.g >= 2:
        for gram in bucket(c, 0xFFF, 3, rng, used):
            used.add(gram)
            add("wrap", short(gram))
            if sl > 1:
                add("one-tag", short(gram, j=1))
    if not has_twins(c) and sl > 1:                      # one tag, many entries: one gram at every j, UNIQUE nodes
        gram = last_home_gram(c) if c.g == 1 else bucket(c, 0xFFE, 1, rng, used)[0]
        used.add(gram)
        add("one-tag", short(gram))
        for x in dict.fromkeys(int(v) for v in random_letters(c, rng, 40)):      # ten UNIQUE nodes under (1, gram)
            if len(roles["one-tag"]) > 10:
                break
            add("one-tag", (x,) + tuple(gram) + rnd(max(0, m - gl - 1)))
        for j in range(2, sl):
            add("one-tag", short(gram, j=j))
    # twins under one tag
    if has_twins(c):
        def pair(top):
            t = (top << 20) | 0x10001
            g2 = solve(c, t, rng, 2, used)
            used.update(g2)
            return g2
        if uniq:
            a, b = pair(0x2A5)
            add("uu", short(a)), add("uu", short(b))
            a, b = pair(0x3B6)
            add("um", short(a)), multi("um", b)
        a, b = pair(0x4C7)
        multi("mm", a), multi("mm", b)
        if sl > 1:
            a, b = pair(0x6E9)
            add("two-j", short(a)), add("two-j", short(b, j=1))
    elif sl > 1:
        gram = fresh()
        multi("two-j", gram), multi("two-j", gram, j=sl - 1)
    # displaced: a foreign tag inserted first into the home slot, then the one UNIQUE j = 0 entry of the target
    if c.g >= 2 and uniq:
        for gram in bucket(c, 0x5C3, 2, rng, used):
            used.add(gram)
            add("displaced", short(gram))
    # run8: eight foreign tags in one home slot, then the target (twins where there are any)
    if c.g >= 2:
        grams = bucket(c, 0x9B7, 9, rng, used)
        used.update(grams)
        for gram in grams[:8]:
            add("run8-foreign", short(gram) if uniq else short(gram, n=m + 1))
        add("run8", short(grams[8]))
        if has_twins(c):
            tw = solve(c, tag_of(c, grams[8]), rng, 1, used)[0]
            used.add(tw)
            multi("run8", tw)
    # MULTI: shared prefix, one long key; 20 bytes and the next whole letter past 20
    multi("shared", fresh())
    add("long", fresh() + rnd(max(m, 30 // L) - gl))
    if m * L <= 20:
        add("k20", fresh() + rnd(20 // L - gl))
    if m <= 20 // L + 1:
        add("k21", fresh() + rnd(20 // L + 1 - gl))
    if L == 4:
        assert all(max(k) > 0xFF for k in keys)
    # near misses: the key's grams, another last letter
    near = []
    for k in keys:
        if len(k) > gl:
            x = k[:-1] + (ctx[(ctx.index(k[-1]) + 1) % len(ctx)] if k[-1] in ctx else ctx[0],)
            if x not in keys:
                near.append(x)
    # decoys: another gram of a key gram's tag, at j = 0, for the tags of every construction above
    key_grams = {k[j:j + gl] for k in keys for j in range(sl) if j + gl <= len(k)}
    decoys = []
    if has_twins(c):
        for role in ("wrap", "uu", "um", "mm", "displaced", "run8"):
            if role not in roles:
                continue
            gram = roles[role][-1][:gl]
            t = tag_of(c, gram)
            try:
                d = solve(c, t, rng, 1, key_grams | used)[0]
            except AssertionError:                      # a one-window gram: both grams of the tag are key grams
                assert c.g == 4
                continue
            used.add(d)
            decoys.append((d, t))
            twins[d] = gram
    return Plan(keys, roles, near, decoys, twins)


# ------------------------------------------------------------------ decoys that pass the bitmap
def _stage1(c, f, grams):
    """(word, bit_a, bit_b) of grams in the single placement's level-1 bitmap (acb_stream_kernel / emul._passes_bitmap)"""
    hw = hash_many(c, grams, 1)
    h1 = hw & np.uint64(M32)
    l1 = f["log2_bits1"]
    n_words = np.uint64(1 << (l1 - 5))
    word = (h1 * n_words) >> np.uint64(32)
    if f["filter_flags"] & emul.FILTER_WIDE:
        a = (hw >> np.uint64(32)) & np.uint64(31)
    else:
        a = (h1 >> np.uint64(32 - l1)) & np.uint64(31)
    return word, a, h1 & np.uint64(31)


def helpers(c, f, decoys, rng):
    """key grams that set the bits each decoy needs in level 1: for the pair placement the decoy with bit 5 of its first
    byte flipped (role 0's word is keyed by bytes 1..3, its bit by the low five bits of byte 0); for the single
    placement grams found in a random sample whose word is the decoy's and whose bits cover one of the decoy's"""
    out = []
    if f["filter_flags"] & emul.FILTER_PAIR:
        for d, _ in decoys:
            out.append((d[0] ^ 0x20,) + tuple(d[1:]))
        return out
    if not decoys:
        return out
    dw, da, db = _stage1(c, f, [d for d, _ in decoys])
    need = [(i, bit) for i in range(len(decoys)) for bit in (da[i], db[i])]
    for _ in range(16):
        P = random_letters(c, rng, (1 << 21, _letters(c)))
        w, a, b = _stage1(c, f, P)
        for i, bit in list(need):
            hit = np.nonzero((w == dw[i]) & ((a == bit) | (b == bit)))[0]
            if len(hit):
                out.append(tuple(int(x) for x in P[hit[0]]))
                need.remove((i, bit))
        if not need:
            return out
    raise AssertionError(f"{c.name}: no helper gram")


def build(c, rng, mp):
    """the plan, its automaton and flat tables: the plan drawn again while the table lacks a property the cell allows
    (a random tag may take a slot first) or has another size than it was planned for, decoy helpers added until the
    level-1 size they were found for stays"""
    lA = 10
    for _ in range(8):
        plan, A, f = _build_once(c, rng, mp, lA)
        if f["log2_anchor_slots"] == lA and capabilities(c) <= properties(c, f, plan):
            break
        lA = f["log2_anchor_slots"]
    return plan, A, f


def _build_once(c, rng, mp, lA):
    plan = build_plan(c, rng, lA)
    base = list(plan.keys)
    log1 = None
    for _ in range(6):
        A = build_automaton(c, plan.keys, mp)
        f = A.flat()
        if f["log2_bits1"] == log1 or not plan.decoys:
            return plan, A, f
        log1 = f["log2_bits1"]
        m = _min_letters(c)
        ctx = kc.ALPHA[c.L] if c.L < 4 else [0x142, 0x1F600]
        extra = [h + tuple(ctx[:1]) * max(0, m - len(h)) for h in helpers(c, f, plan.decoys, rng)]
        plan.keys = base + [k for k in dict.fromkeys(extra) if k not in base]
    raise AssertionError(f"{c.name}: level 1 does not settle")


def pkg_key(c, k):
    if c.seq:
        return tuple(k)
    return kc._pkg_key(k, c.L)


def build_automaton(c, keys, mp):
    if not c.seq:
        return kc._build(c.cell, keys, mp)
    import pyahocorasick_b200 as ac
    mod = ac.flavour("unicode")
    A = mod.Automaton(mod.STORE_INTS, mod.KEY_SEQUENCE)
    for i, k in enumerate(keys):
        A.add_word(tuple(k), i)
    with mp.context() as m:
        m.setenv("ACB_FILTER", c.env)
        m.delenv("ACB_FORCE_TAGMAP", raising=False)
        A.make_automaton()
    return A


# ------------------------------------------------------------------ the table, read back
@dataclasses.dataclass
class Entry:
    slot: int
    tag: int
    kid: int
    j: int
    len: int
    last: bool
    raw: bytes


def entries(f):
    A = np.asarray(f["anchors"]).reshape(-1, 8).astype(np.uint32)
    out = []
    for slot in np.nonzero(A[:, 0])[0]:
        e = A[slot]
        raw = b"".join(int(w).to_bytes(4, "little") for w in e[3:8])
        out.append(Entry(int(slot), int(e[0]), int(np.int32(e[1])), int(e[2]) & 0xFF, (int(e[2]) >> 8) & 0xFF,
                         bool((int(e[2]) >> 16) & 1), raw))
    return out


def chain(f, tag):
    """the slots a lookup of `tag` visits (home slot on, wrapping) and the tag's own entries among them, in order"""
    A = np.asarray(f["anchors"]).reshape(-1, 8)
    lA = f["log2_anchor_slots"]
    mask = (1 << lA) - 1
    slot, visited, own = tag >> (32 - lA), [], []
    for _ in range(mask + 1):
        e = A[slot]
        if int(e[0]) == 0:
            break
        visited.append(slot)
        if int(e[0]) == tag:
            own.append(slot)
            if (int(e[2]) >> 16) & 1:
                break
        slot = (slot + 1) & mask
    return visited, own


def entry_gram(c, e):
    """the gram an entry stands for: MULTI entries carry it, UNIQUE ones carry the key from its start"""
    return e.raw[:c.g] if e.kid < 0 else e.raw[e.j:e.j + c.g]


def properties(c, f, plan):
    """the properties the table has, read from f["anchors"]: what the kernels' walks will meet"""
    E = entries(f)
    lA = f["log2_anchor_slots"]
    mask = (1 << lA) - 1
    by_tag = {}
    for e in E:
        by_tag.setdefault(e.tag, []).append(e)
    have = set()
    kid = {k: i for i, k in enumerate(plan.keys)}
    for t, es in by_tag.items():
        visited, own = chain(f, t)
        home = t >> (32 - lA)
        assert sorted(own) == sorted(e.slot for e in es), (hex(t), own, [e.slot for e in es])   # every entry reachable
        assert sum(e.last for e in es) == 1 and E[[x.slot for x in E].index(own[-1])].last
        if any(s < home for s in own):
            have.add("wrap")                            # an entry past the last slot
            if any(s >= home for s in own):
                have.add("wrap-split")                  # one tag's entries on both sides of it
        grams = {(entry_gram(c, e), e.kid < 0) for e in es}
        distinct = {g for g, _ in grams}
        uniq = [e for e in es if e.kid >= 0]
        mult = [e for e in es if e.kid < 0]
        if len(distinct) > 1:
            for x in uniq:
                for y in uniq:
                    if x.j == y.j and entry_gram(c, x) != entry_gram(c, y):
                        have.add("uu")
                for y in mult:
                    if entry_gram(c, x) != entry_gram(c, y):
                        have.add("um")
            if len({entry_gram(c, e) for e in mult}) > 1:
                have.add("mm")
        elif len(mult) > 1:
            have.add("mm")                              # one gram, MULTI at two j
        if len({e.j for e in es}) > 1:
            have.add("two-j")
        if len(distinct) == 1 and len(es) >= 3:
            have.add("one-tag")
        first = visited.index(own[0])
        if len(es) == 1 and uniq and es[0].j == 0 and first >= 1:
            have.add("displaced")
        if first >= 8:
            have.add("run8")
    for role, want in (("shared", lambda e: e.kid < 0), ("long", lambda e: e.kid < 0),
                       ("k20", lambda e: e.kid >= 0 and e.len == 20), ("k21", lambda e: e.kid < 0)):
        for k in plan.roles.get(role, ()):
            t = tag_of(c, k[:_letters(c)])
            hits = [e for e in by_tag.get(t, ()) if e.j == 0 and entry_gram(c, e) == bytes(_bytes(c, k[:_letters(c)])) and want(e)]
            if role == "k20":
                hits = [e for e in hits if e.kid == kid[k]]
            if hits:
                have.add(role)
    return have


# ------------------------------------------------------------------ texts
Item = collections.namedtuple("Item", "start n kind")      # in letters; kind: key, near, decoy


def zone(c, f, plan, rng):
    """every key, near miss and decoy, first back to back (one dense run: consecutive candidates of one warp turn take
    different ways through the table), then each followed by filler; decoys start at a probe position (an even one for
    the pair placement: role 0, whose level-1 bit the helpers set)"""
    L = c.L
    align = max(c.s, 2 if f["filter_flags"] & emul.FILTER_PAIR else 1)
    keys, near, dec = plan.keys, plan.near, [d for d, _ in plan.decoys]
    mixed = []
    for i in range(max(len(keys), len(near), 4 * len(dec))):
        for kind, lst in (("key", keys), ("near", near), ("decoy", dec)):
            if lst:
                mixed.append((kind, lst[i % len(lst)]))
    out, items = [], []

    def fill(n):
        out.extend(int(x) for x in rng.choice(kc.ALPHA[L], size=n))

    for dense in (True, False):
        for kind, k in mixed:
            if kind == "decoy":
                fill((-len(out) * L) % align // L)
            items.append(Item(len(out), len(k), kind))
            out.extend(k)
            if not dense:
                fill(1 + int(rng.integers(0, 2 * c.s // L + 2)))
    return np.asarray(out, dtype=np.int64), items


def text(c, f, plan, rng, n_bytes):
    """n_bytes of kernel_cells._text (the keys across every lane run, slice and tile boundary), the zone from its start
    and a key on its last letters; returns the letters and the zone's items"""
    t, _ = kc._text(c.cell, plan.keys, rng, n_bytes)
    z, items = zone(c, f, plan, rng)
    assert z.size + 64 < t.size, (z.size, t.size)
    t[:z.size] = z
    k = plan.roles["wrap" if "wrap" in plan.roles else "long"][0]
    t[t.size - len(k):] = k
    items.append(Item(t.size - len(k), len(k), "key"))
    return t.astype(np.int64), items


def ragged(c, rng, n, items):
    """offsets (letters) whose haystacks start at item starts, end at item ends and cut through items (a cut between
    an item's start and its probe, and between its probe and its end), plus random cuts and runs of empty haystacks"""
    cuts = [rng.integers(0, n + 1, size=60)]
    for i, it in enumerate(items):
        r = i % 3
        if r == 0:
            cuts.append([it.start])
        elif r == 1:
            cuts.append([it.start + it.n])
        elif it.n > 1:
            cuts.append([it.start + 1 + (i // 3) % (it.n - 1)])
    cuts = np.sort(np.concatenate([np.asarray(x, dtype=np.int64) for x in cuts]))
    cuts = np.concatenate([cuts, cuts[::13], cuts[::13], cuts[4::29]])
    return np.concatenate([[0, 0], np.sort(np.clip(cuts, 0, n)), [n, n]]).astype(np.int64)
