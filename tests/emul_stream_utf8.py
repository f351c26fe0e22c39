"""A Python restatement of how a UTF-8 stream batch stages a feed (DESIGN section 4.21), on top of emul_utf8.

Each stream carries the bytes of a letter its text has not finished.  A chunk is staged as carry || chunk without its
new held tail: the bytes from the last non-continuation byte among the last 3 to the end, when that byte's maximal
valid prefix runs to the end and is shorter than its sequence -- with one exception CPython makes: ED followed by A0-BF
(the start of an encoded surrogate) is held too, and decodes as two invalid letters once a third byte or the end
arrives.  A final stage (finish) holds nothing back, so a truncated prefix decodes as the end of a haystack does."""
import emul_utf8 as eu


def hold(x: bytes) -> int:
    """the bytes at the end of x that begin an unfinished letter (0 to 3)"""
    for p in range(len(x) - 1, max(len(x) - 3, 0) - 1, -1):
        if x[p] in eu.CONT:
            continue
        d = len(x) - p
        if x[p] == 0xED and d == 2:                        # CPython keeps ED A0-BF too, until a third byte shows it invalid
            return d
        k, whole = eu.prefix(x, p)
        return d if k == d and not whole and eu._lead(x[p])[1] > d else 0
    return 0


def stage(carry: bytes, chunk: bytes, final: bool = False):
    """(the staged haystack, the new carry) of a chunk fed behind `carry`"""
    x = carry + chunk
    k = 0 if final else hold(x)
    return x[:len(x) - k], x[len(x) - k:]
