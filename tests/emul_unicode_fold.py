"""Unicode case-insensitive matching restated (find_all_batch(..., case_insensitive=True) and the leftmost and
replacement methods with it): the fold, the groups of keys that fold to one text, and the definitions the GPU is checked
against.  Letters are ints (code points, or latin-1 byte values); keys are given as a list indexed by key id, None for a
removed id.  The alias expansion is emul_fold.expand, which does not depend on the fold.  Not a test module."""
import functools

import numpy as np

from emul_fold import expand  # noqa: F401  (the expansion of this fold's alias lists, restated once)
from emul_replace import definition as replaced
from emul_words import definition as whole_words


def simple_fold(c: int) -> int:
    """Unicode simple case folding of one code point: a one-letter casefold(), else a one-letter lower(), else itself"""
    ch = chr(c)
    for f in (ch.casefold(), ch.lower()):
        if len(f) == 1:
            return ord(f)
    return c


@functools.lru_cache(maxsize=None)
def canonical() -> np.ndarray:
    """int64[0x110000]: each code point's canonical letter, the lowest code point of equal simple_fold"""
    sf = np.fromiter((simple_fold(c) for c in range(0x110000)), dtype=np.int64, count=0x110000)
    order = np.lexsort((np.arange(0x110000), sf))          # by fold value, then code point: each class's minimum first
    first = np.ones(0x110000, dtype=bool)
    first[1:] = sf[order][1:] != sf[order][:-1]
    low = np.maximum.accumulate(np.where(first, np.arange(0x110000), 0))
    out = np.empty(0x110000, dtype=np.int64)
    out[order] = order[low]
    return out


def fold(letters):
    """the letters folded: code points to their canonical letter, values above 0x10FFFF kept"""
    a = np.asarray(letters, dtype=np.int64)
    inside = a < 0x110000
    return np.where(inside, canonical()[np.where(inside, a, 0)], a)


def groups(keys):
    """(rep, aliases): rep[id] = the lowest id whose key folds to the same text, for every live id; aliases[r] = the other
    ids of representative r's group, ascending"""
    first, rep, aliases = {}, {}, {}
    for kid, k in enumerate(keys):
        if k is None:
            continue
        r = first.setdefault(tuple(fold(k).tolist()), kid)
        rep[kid] = r
        if r != kid:
            aliases.setdefault(r, []).append(kid)
    return rep, aliases


def find_all(keys, hays):
    """every (hay, end, key id) whose folded key equals the folded text ending at end, in the reference order with
    ascending id among keys of one length"""
    out = []
    fk = [None if k is None else fold(k).tolist() for k in keys]
    for h, hay in enumerate(hays):
        fh = fold(hay).tolist()
        for e in range(len(fh)):
            here = [(-len(k), kid) for kid, k in enumerate(fk) if k and len(k) <= e + 1 and fh[e + 1 - len(k):e + 1] == k]
            out += [(h, e, kid) for _, kid in sorted(here)]
    return out


def leftmost(keys, hays, first: bool, is_word=None):
    """the leftmost-first (first=True) or leftmost-longest selection over the folded matches of the representatives,
    whole words only when is_word is given (tested in the text as given)"""
    rep, _ = groups(keys)
    kl = [0 if k is None else len(k) for k in keys]
    full = [r for r in find_all(keys, hays) if rep[r[2]] == r[2]]
    if is_word is not None:
        full = whole_words(hays, full, kl, is_word)
    out = []
    for h in range(len(hays)):
        cand = sorted((e - kl[k] + 1, k if first else -kl[k], e, k) for hh, e, k in full if hh == h)
        p = 0
        for s, _, e, k in cand:
            if s >= p:
                out.append((h, e, k))
                p = e + 1
    return out


def replace(keys, reps, hays, first: bool, is_word=None):
    """each haystack with the matches `leftmost` chooses replaced by reps[key id], every other letter as given"""
    chosen = leftmost(keys, hays, first, is_word)
    kl = [0 if k is None else len(k) for k in keys]
    return [replaced(hay, [(e, k) for hh, e, k in chosen if hh == h], kl, reps) for h, hay in enumerate(hays)]
