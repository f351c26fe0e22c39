"""A Python restatement of the per-byte UTF-8 rule the GPU decodes by (DESIGN section 4.20), independent of the library.

A byte starts a letter unless it is a continuation byte (0x80-0xBF) that the nearest non-continuation byte at most 3
bytes before it covers with its maximal valid prefix.  The maximal valid prefix follows Unicode Table 3-7: the second
byte is narrowed after E0 (A0-BF), ED (80-9F), F0 (90-BF) and F4 (80-8F); C0, C1 and F5-FF never lead; it never crosses
the end of the haystack.  A letter whose maximal prefix is not a whole sequence is U+FFFD; the first such letter is the
strict error, from its first byte to the end of its prefix."""

CONT = range(0x80, 0xC0)


def _lead(b):
    """(second-byte range, sequence length) of a lead byte, or (None, 1) for a byte that leads nothing"""
    if b < 0x80:
        return None, 1
    if 0xC2 <= b <= 0xDF:
        return (0x80, 0xBF), 2
    if 0xE0 <= b <= 0xEF:
        return ((0xA0, 0xBF) if b == 0xE0 else (0x80, 0x9F) if b == 0xED else (0x80, 0xBF)), 3
    if 0xF0 <= b <= 0xF4:
        return ((0x90, 0xBF) if b == 0xF0 else (0x80, 0x8F) if b == 0xF4 else (0x80, 0xBF)), 4
    return None, 0


def prefix(h: bytes, i: int):
    """(length of the maximal valid prefix at byte i, whether it is a whole sequence)"""
    rng, need = _lead(h[i])
    if need == 1:
        return 1, True
    if need == 0:
        return 1, False
    k = 1
    while k < need and i + k < len(h):
        lo, hi = rng if k == 1 else (0x80, 0xBF)
        if not lo <= h[i + k] <= hi:
            break
        k += 1
    return k, k == need


def starts(h: bytes):
    """the bytes of h that start a letter, each decided from at most 3 bytes before it"""
    out = []
    for i, c in enumerate(h):
        start = True
        if c in CONT:
            for d in (1, 2, 3):
                j = i - d
                if j < 0:
                    break
                if h[j] in CONT:
                    continue
                start = prefix(h, j)[0] <= d
                break
        if start:
            out.append(i)
    return out


def letters(h: bytes):
    """the code points h decodes to under "replace" (U+FFFD per invalid letter)"""
    out = []
    for s in starts(h):
        k, ok = prefix(h, s)
        out.append(ord(h[s:s + k].decode("utf-8")) if ok else 0xFFFD)
    return out


def decode(h: bytes) -> str:
    return "".join(map(chr, letters(h)))


def first_error(h: bytes):
    """(start, end) of the first invalid letter, or None"""
    for s in starts(h):
        k, ok = prefix(h, s)
        if not ok:
            return s, s + k
    return None
