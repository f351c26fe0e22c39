"""ASCII case-insensitive matching restated (find_all_batch(..., ascii_case_insensitive=True) and the leftmost and
replacement methods with it): the fold, the groups of keys that fold to one text, the device's alias expansion, and the
definitions the GPU is checked against.  Letters are ints (byte values or code points); keys are given as a list indexed
by key id, None for a removed id.  Not a test module."""
import numpy as np

from emul_replace import definition as replaced
from emul_words import definition as whole_words


def fold(letters):
    """the letters with 0x41..0x5A made small: the whole letter value is compared, nothing else changes"""
    a = np.asarray(letters, dtype=np.int64)
    return np.where((a >= 0x41) & (a <= 0x5A), a + 0x20, a)


def fold_swar(words: np.ndarray) -> np.ndarray:
    """the fold kernel's 1-byte-letter formula on uint32 words of four bytes (acb_device.cu, fold_bytes)"""
    x = np.asarray(words, dtype=np.uint32)
    h = x & np.uint32(0x7F7F7F7F)
    upper = (h + np.uint32(0x3F3F3F3F)) & ~(h + np.uint32(0x25252525)) & ~x & np.uint32(0x80808080)
    return x | (upper >> np.uint32(2))


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


def alias_csr(keys):
    """the alias lists as acb_table_upload_folded takes them: (alias_ptr over 1 + the largest representative, alias_ids)"""
    rep, aliases = groups(keys)
    ptr = np.zeros(max(rep.values()) + 2, dtype=np.int64)
    for r, ids in aliases.items():
        ptr[r + 1] = len(ids)
    return np.cumsum(ptr), np.array([k for r in sorted(aliases) for k in aliases[r]], dtype=np.int64)


def expand(rec: np.ndarray, alias_ptr: np.ndarray, alias_ids: np.ndarray, cap: int):
    """acb_expand_aliases_device over (n, 3) records: count per record, exclusive sum, scatter -> (stored records, total)"""
    rec = np.asarray(rec, dtype=np.int64).reshape(-1, 3)
    k = rec[:, 2]
    inside = k < len(alias_ptr) - 1
    cnt = np.ones(len(rec), dtype=np.int64)
    cnt[inside] += alias_ptr[k[inside] + 1] - alias_ptr[k[inside]]
    pos = np.cumsum(cnt) - cnt
    total = int(cnt.sum())
    out = np.zeros((total, 3), dtype=np.int64)
    for i in range(len(rec)):
        out[pos[i]] = rec[i]
        if inside[i]:
            for j, a in enumerate(alias_ids[alias_ptr[k[i]]:alias_ptr[k[i] + 1]].tolist()):
                out[pos[i] + 1 + j] = (rec[i, 0], rec[i, 1], a)
    return out[:cap], total


def find_all(keys, hays):
    """every (hay, end, key id) whose key equals the folded text ending at end, in the reference order with ascending id
    among keys of one length"""
    out = []
    fk = [None if k is None else fold(k).tolist() for k in keys]
    for h, hay in enumerate(hays):
        fh = fold(hay).tolist()
        for e in range(len(fh)):
            here = [(-len(k), kid) for kid, k in enumerate(fk) if k and len(k) <= e + 1 and fh[e + 1 - len(k):e + 1] == k]
            out += [(h, e, kid) for _, kid in sorted(here)]
    return out


def key_lengths(keys):
    return [0 if k is None else len(k) for k in keys]


def leftmost(keys, hays, first: bool, is_word=None):
    """the leftmost-first (first=True) or leftmost-longest selection over the folded matches of the representatives,
    whole words only when is_word is given (tested in the text as given)"""
    rep, _ = groups(keys)
    kl = key_lengths(keys)
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
    kl = key_lengths(keys)
    return [replaced(hay, [(e, k) for hh, e, k in chosen if hh == h], kl, reps) for h, hay in enumerate(hays)]
