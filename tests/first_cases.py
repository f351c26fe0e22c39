"""The leftmost-first rule's independent oracle: Python's `re`, shared by the leftmost-first tests.  Not a test module.

An alternation of the escaped keys in key-id order, scanned with finditer, is leftmost-first non-overlapping matching:
the leftmost position where some alternative matches, the first alternative that matches there, then on after it.
Whole words wrap it in (?<![W])(?:...)(?![W]) with W the word letters as an explicit class, so a haystack edge counts as
a non-word letter.  Replacement is pattern.sub with each key's replacement."""
import re

from batch_cases import CASES


def _text(case, letters):
    """letters as `re` takes them: bytes for the bytes flavour, else str"""
    fl = CASES[case][0]
    return bytes(letters) if fl == "bytes" else "".join(map(chr, letters))


def pattern(case, keys, word_letters=None):
    """the alternation of keys (letter lists, in key-id order); word_letters: the whole-word form, with these letters
    (an iterable of letter values) as W"""
    alt = [re.escape(_text(case, k)) for k in keys]
    bytes_flavour = CASES[case][0] == "bytes"
    body = (b"|" if bytes_flavour else "|").join(alt)
    if word_letters is None:
        return re.compile(body)
    w = sorted(set(word_letters))
    cls = "".join(f"\\x{c:02x}" if c < 256 else f"\\U{c:08x}" for c in w)
    if bytes_flavour:
        cls = cls.encode()
        return re.compile(b"(?<![" + cls + b"])(?:" + body + b")(?![" + cls + b"])") if w else re.compile(body)
    return re.compile("(?<![" + cls + "])(?:" + body + ")(?![" + cls + "])") if w else re.compile(body)


def find(case, keys, hays, word_letters=None):
    """[(hay, end, key id)] of the leftmost-first matches of every haystack"""
    p = pattern(case, keys, word_letters)
    ids = {_text(case, k): i for i, k in enumerate(keys)}
    out = []
    for h, letters in enumerate(hays):
        for m in p.finditer(_text(case, letters)):
            out.append((h, m.end() - 1, ids[m.group()]))
    return out


def sub(case, keys, reps, hays, word_letters=None):
    """every haystack with its leftmost-first matches replaced (reps: letter lists by key id), as letter lists"""
    p = pattern(case, keys, word_letters)
    rep = {_text(case, k): _text(case, r) for k, r in zip(keys, reps)}
    out = []
    for letters in hays:
        t = p.sub(lambda m: rep[m.group()], _text(case, letters))
        out.append(list(t) if isinstance(t, bytes) else [ord(c) for c in t])
    return out


def np_greedy_first(full, key_len):
    """the leftmost-first definition over a full record array (hay_id, end_index, key_id), vectorised but for the walk
    itself -> int64 rows (hay, end, key) in haystack order, then end ascending"""
    import numpy as np
    if len(full) == 0:
        return np.empty((0, 3), dtype=np.int64)
    hay, end, key = (np.asarray(full[f]).astype(np.int64) for f in ("hay_id", "end_index", "key_id"))
    ln = np.asarray(key_len, dtype=np.int64)[key]
    start = end - ln + 1
    o = np.lexsort((key, start, hay))
    hay, start, ln, end, key = hay[o], start[o], ln[o], end[o], key[o]
    first = np.ones(len(o), dtype=bool)
    first[1:] = (hay[1:] != hay[:-1]) | (start[1:] != start[:-1])
    hay, start, ln, end, key = hay[first], start[first], ln[first], end[first], key[first]
    flat = hay * (np.int64(1) << 32) + start                 # start + len < 2^32: one sortable number per (hay, start)
    nxt = np.searchsorted(flat, flat + ln)
    ok = nxt < len(flat)
    ok[ok] = hay[nxt[ok]] == hay[ok]
    nx = np.where(ok, nxt, -1).tolist()
    chosen = []
    for i in np.nonzero(np.r_[True, hay[1:] != hay[:-1]])[0].tolist():
        while i >= 0:
            chosen.append(i)
            i = nx[i]
    chosen = np.array(sorted(chosen), dtype=np.int64)
    return np.stack([hay[chosen], end[chosen], key[chosen]], axis=1)
