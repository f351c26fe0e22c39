"""pyahocorasick_b200 -- H100-native Aho-Corasick batch search behind the
``ahocorasick.Automaton`` API of WojciechMula/pyahocorasick.

    import pyahocorasick_b200 as ahocorasick

The module mirrors the reference's module surface (src/pyahocorasick.c:67-137):
``Automaton``, the ``EMPTY/TRIE/AHOCORASICK``, ``STORE_*``, ``KEY_*``, ``MATCH_*`` constants and the
``unicode`` flag.  Like the reference, the flavour is chosen by the environment variables
``AHOCORASICK_BYTES`` / ``AHOCORASICK_UNICODE`` (setup.py:17-34; default = unicode) -- here at import
time rather than build time -- and ``flavour("bytes"|"unicode")`` gives either flavour explicitly.

Every search (``iter``, ``find_all``, ``find_all_batch``) runs on the GPU through the C ABI in
``include/acb200.h``; there is no CPU search path and no fallback.
"""
from __future__ import annotations

import os
import types

from . import automaton as _a
from . import serialize as _serialize
from .automaton import (AHOCORASICK, EMPTY, KEY_SEQUENCE, KEY_STRING, MATCH_AT_LEAST_PREFIX,  # noqa: F401
                        MATCH_AT_MOST_PREFIX, MATCH_EXACT_LENGTH, STORE_ANY, STORE_INTS, STORE_LENGTH,
                        TRIE, AutomatonSearchIter, Matches, load)

__version__ = "0.1.0"


class _UnicodeAutomaton(_a.Automaton):
    """str keys and haystacks (the reference's default build)."""
    _UNICODE = True


class _BytesAutomaton(_a.Automaton):
    """bytes keys and haystacks (the reference built with AHOCORASICK_BYTES)."""
    _UNICODE = False


_UnicodeAutomaton.__name__ = _UnicodeAutomaton.__qualname__ = "Automaton"
_BytesAutomaton.__name__ = _BytesAutomaton.__qualname__ = "Automaton"

_CONSTS = dict(EMPTY=EMPTY, TRIE=TRIE, AHOCORASICK=AHOCORASICK, STORE_INTS=STORE_INTS, STORE_LENGTH=STORE_LENGTH,
               STORE_ANY=STORE_ANY, KEY_STRING=KEY_STRING, KEY_SEQUENCE=KEY_SEQUENCE,
               MATCH_EXACT_LENGTH=MATCH_EXACT_LENGTH, MATCH_AT_MOST_PREFIX=MATCH_AT_MOST_PREFIX,
               MATCH_AT_LEAST_PREFIX=MATCH_AT_LEAST_PREFIX, load=load)
_flavours = {}


def flavour(name: str):
    """A module-like namespace for one flavour: ``flavour("bytes").Automaton`` ..."""
    if name not in ("bytes", "unicode"):
        raise ValueError("flavour must be 'bytes' or 'unicode'")
    if name not in _flavours:
        m = types.SimpleNamespace(**_CONSTS)
        m.unicode = 1 if name == "unicode" else 0
        m.Automaton = _UnicodeAutomaton if name == "unicode" else _BytesAutomaton
        m.load = (lambda cls: lambda *args: _serialize.load(cls, *args))(m.Automaton)
        _flavours[name] = m
    return _flavours[name]


if "AHOCORASICK_BYTES" in os.environ and "AHOCORASICK_UNICODE" in os.environ:
    raise ImportError("only one of AHOCORASICK_UNICODE and AHOCORASICK_BYTES may be set")
unicode = 0 if "AHOCORASICK_BYTES" in os.environ else 1
Automaton = flavour("unicode" if unicode else "bytes").Automaton
