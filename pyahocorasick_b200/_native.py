"""ctypes binding of include/acb200.h (libacb200.so).  No fallback: if the native
library is missing or has no usable device, the search entry points raise."""
from __future__ import annotations

import ctypes
import os

import numpy as np

_PKG = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("ACB_LIB") or os.path.join(_PKG, "_native", "libacb200.so")   # ACB_LIB: experimental builds

ABI_VERSION = 5            # ACB_ABI_VERSION of include/acb200.h this binding was written against
ACB_OK, ACB_ENOMEM, ACB_EINVAL, ACB_ESTATE, ACB_ECUDA, ACB_EOVERFLOW, ACB_ERANGE = 0, -1, -2, -3, -4, -5, -6
ALGO_AUTO, ALGO_FILTER, ALGO_DFA, ALGO_LONG = 0, 1, 2, 3
ALGOS = {"auto": ALGO_AUTO, "filter": ALGO_FILTER, "dfa": ALGO_DFA, "long": ALGO_LONG}
SELECT_LONGEST, SELECT_FIRST = 0, 1     # ACB_SELECT_*: the match a leftmost selection takes at a start
MAX_SKIP = 1024            # ACB_MAX_SKIP: largest skip set of the white-space scans
UTF8_STRICT, UTF8_REPLACE = 0, 1        # ACB_UTF8_*: the errors kind of acb_utf8_decode_device

MATCH_DTYPE = np.dtype([("hay_id", "<i4"), ("end_index", "<i4"), ("key_id", "<i4")])


class FlatView(ctypes.Structure):
    _fields_ = [
        ("n_states", ctypes.c_int32), ("n_classes", ctypes.c_int32), ("n_keys", ctypes.c_int32),
        ("letter_bytes", ctypes.c_int32), ("min_key_bytes", ctypes.c_int32), ("max_key_bytes", ctypes.c_int32),
        ("byte_class", ctypes.POINTER(ctypes.c_uint8)),
        ("goto_cm", ctypes.POINTER(ctypes.c_int32)), ("fail", ctypes.POINTER(ctypes.c_int32)),
        ("letter_fail", ctypes.POINTER(ctypes.c_int32)),
        ("key_of", ctypes.POINTER(ctypes.c_int32)), ("out_ptr", ctypes.POINTER(ctypes.c_int32)),
        ("out_idx", ctypes.POINTER(ctypes.c_int32)), ("key_len", ctypes.POINTER(ctypes.c_int32)),
        ("gram_bytes", ctypes.c_int32), ("stride", ctypes.c_int32),
        ("log2_bits1", ctypes.c_int32), ("log2_anchor_slots", ctypes.c_int32), ("log2_bits3", ctypes.c_int32),
        ("bitmap1", ctypes.POINTER(ctypes.c_uint32)), ("bitmap3", ctypes.POINTER(ctypes.c_uint32)),
        ("anchors", ctypes.POINTER(ctypes.c_uint32)),
        ("filter_flags", ctypes.c_int32), ("log2_bits2", ctypes.c_int32),
    ]


class NativeError(RuntimeError):
    pass


_lib = None


def lib() -> ctypes.CDLL:
    """Load libacb200.so (built by `python -m pyahocorasick_b200.build`)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing: build it with `python -m pyahocorasick_b200.build` "
            "(nvcc, sm_90a).  There is no CPU fallback.")
    L = ctypes.CDLL(LIB_PATH)
    vp, i32, i64 = ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64
    pi32, pi64 = ctypes.POINTER(ctypes.c_int32), ctypes.POINTER(ctypes.c_int64)
    sig = {
        "acb_trie_new": (vp, [ctypes.c_int]),
        "acb_trie_free": (None, [vp]),
        "acb_trie_clear": (ctypes.c_int, [vp]),
        "acb_trie_add_word": (ctypes.c_int, [vp, vp, i64, i32, pi32]),
        "acb_trie_remove_word": (ctypes.c_int, [vp, vp, i64, pi32]),
        "acb_trie_find": (ctypes.c_int, [vp, vp, i64, pi32, pi32]),
        "acb_trie_longest_prefix": (i64, [vp, vp, i64]),
        "acb_trie_make_automaton": (ctypes.c_int, [vp, pi32]),
        "acb_trie_kind": (ctypes.c_int, [vp]),
        "acb_trie_count": (i64, [vp]),
        "acb_trie_longest_word": (i64, [vp]),
        "acb_trie_nodes": (i64, [vp]),
        "acb_trie_links": (i64, [vp]),
        "acb_trie_host_bytes": (i64, [vp]),
        "acb_trie_key_order": (ctypes.c_int, [vp, vp, i64, pi64]),
        "acb_trie_key_ranges": (ctypes.c_int, [vp, vp, vp, vp, vp, vp, pi64]),
        "acb_trie_content_hash": (ctypes.c_uint64, [vp]),
        "acb_trie_flat_save": (ctypes.c_int, [vp, vp, i64, ctypes.POINTER(i64)]),
        "acb_trie_flat_load": (ctypes.c_int, [vp, vp, i64]),
        "acb_trie_flat_view": (ctypes.c_int, [vp, ctypes.POINTER(FlatView)]),
        "acb_trie_export_nodes": (ctypes.c_int, [vp, ctypes.c_int, vp, i64, vp, i64, pi64, pi64, vp, vp, i64]),
        "acb_trie_import_nodes": (ctypes.c_int, [vp, vp, i64, i64, ctypes.c_int, ctypes.c_int, ctypes.c_int, vp, vp, i64, pi64, pi64,
                                                 vp, i64, vp, pi64]),
        "acb_node_records_span": (ctypes.c_int, [vp, i64, i64, ctypes.c_int, pi64]),
        "acb_device_count": (ctypes.c_int, [pi32]),
        "acb_table_upload": (ctypes.c_int, [vp, ctypes.c_int, ctypes.POINTER(vp)]),
        "acb_table_free": (None, [vp]),
        "acb_table_device_bytes": (i64, [vp]),
        "acb_scan_geometry": (ctypes.c_int, [ctypes.c_int, pi32, i32]),          # test hooks (acb200.h)
        "acb_table_set_cta_limit": (ctypes.c_int, [vp, i32]),
        "acb_table_scan_grid": (ctypes.c_int, [vp, i64, pi32, pi64]),
        "acb_scan_device": (ctypes.c_int, [vp, vp, i64, vp, i64, i64, vp, i64, vp, vp, ctypes.c_int]),
        "acb_scan_host": (ctypes.c_int, [vp, vp, i64, vp, i64, i64, vp, i64, pi64, ctypes.c_int, ctypes.c_int]),
        "acb_copy_records": (ctypes.c_int, [vp, vp, i64]),
        "acb_take_records": (ctypes.c_int, [vp, ctypes.POINTER(vp), pi64, pi64]),
        "acb_release_records": (None, [vp, i64]),
        "acb_sort_matches_device": (ctypes.c_int, [vp, vp, i64, i64, i64, vp]),
        "acb_table_set_long_state": (ctypes.c_int, [vp, ctypes.c_int32]),
        "acb_table_get_long_state": (ctypes.c_int, [vp, ctypes.POINTER(ctypes.c_int32)]),
        "acb_streams_new": (ctypes.c_int, [vp, i64, ctypes.c_int, ctypes.POINTER(vp)]),
        "acb_streams_free": (None, [vp]),
        "acb_streams_reset": (ctypes.c_int, [vp, vp, i64]),
        "acb_streams_feed_device": (ctypes.c_int, [vp, vp, vp, i64, vp, i64, i64, vp, vp, i64, vp, vp, ctypes.c_int]),
        "acb_streams_feed_host": (ctypes.c_int, [vp, vp, vp, i64, vp, i64, i64, vp, vp, i64, pi64, ctypes.c_int, ctypes.c_int]),
        "acb_streams_positions": (ctypes.c_int, [vp, vp, i64]),
        "acb_space_letters": (ctypes.c_int, [ctypes.c_int, ctypes.c_int, vp, i64, pi64]),
        "acb_scan_device_skip": (ctypes.c_int, [vp, vp, i64, vp, i64, i64, vp, i64, vp, vp, ctypes.c_int, vp, i64]),
        "acb_scan_host_skip": (ctypes.c_int, [vp, vp, i64, vp, i64, i64, vp, i64, pi64, ctypes.c_int, ctypes.c_int, vp, i64]),
        "acb_streams_new_skip": (ctypes.c_int, [vp, i64, vp, i64, ctypes.POINTER(vp)]),
        "acb_last_skip_ms": (ctypes.c_int, [ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_float)]),
        "acb_lookup_device": (ctypes.c_int, [vp, vp, i64, vp, i64, i64, vp, vp, vp]),
        "acb_lookup_host": (ctypes.c_int, [vp, vp, i64, vp, i64, i64, vp, vp]),
        "acb_table_upload_key_ranges": (ctypes.c_int, [vp, vp]),
        "acb_select_device": (ctypes.c_int, [vp, vp, i64, vp, i64, i64, i64, ctypes.c_int, vp, vp, i64, vp, vp]),
        "acb_select_host": (ctypes.c_int, [vp, vp, i64, vp, i64, i64, i64, ctypes.c_int, vp, vp, i64, pi64]),
        "acb_leftmost_longest_device": (ctypes.c_int, [vp, vp, i64, i64, i64, vp, i64, vp, vp]),
        "acb_scan_host_leftmost": (ctypes.c_int, [vp, vp, i64, vp, i64, i64, vp, i64, pi64, ctypes.c_int]),
        "acb_last_leftmost_ms": (ctypes.c_int, [ctypes.POINTER(ctypes.c_float), i32]),
        "acb_leftmost_first_device": (ctypes.c_int, [vp, vp, i64, i64, i64, vp, i64, vp, vp]),
        "acb_scan_host_leftmost_kind": (ctypes.c_int, [vp, ctypes.c_int, vp, i64, vp, i64, i64, vp, i64, vp, i64, pi64,
                                                       ctypes.c_int]),
        "acb_replacer_new_kind": (ctypes.c_int, [vp, ctypes.c_int, vp, i64, vp, i64, ctypes.POINTER(vp)]),
        "acb_streams_new_leftmost_kind": (ctypes.c_int, [vp, i64, ctypes.c_int, vp, i64, ctypes.POINTER(vp)]),
        "acb_replacer_new": (ctypes.c_int, [vp, vp, i64, vp, i64, ctypes.POINTER(vp)]),
        "acb_replacer_free": (None, [vp]),
        "acb_replace_device": (ctypes.c_int, [vp, vp, vp, i64, vp, i64, i64, vp, i64, vp, vp, vp, i64, vp, vp]),
        "acb_replace_host": (ctypes.c_int, [vp, vp, vp, i64, vp, i64, i64, ctypes.c_int, vp, vp, i64, pi64]),
        "acb_last_replace_ms": (ctypes.c_int, [ctypes.POINTER(ctypes.c_float), i32]),
        "acb_streams_new_leftmost": (ctypes.c_int, [vp, i64, ctypes.POINTER(vp)]),
        "acb_streams_feed_leftmost_device": (ctypes.c_int, [vp, vp, vp, i64, vp, i64, i64, vp, ctypes.c_int, vp, i64, vp, vp,
                                                            ctypes.c_int]),
        "acb_streams_feed_leftmost_host": (ctypes.c_int, [vp, vp, vp, i64, vp, i64, i64, vp, ctypes.c_int, vp, i64, pi64,
                                                          ctypes.c_int]),
        "acb_streams_replace_device": (ctypes.c_int, [vp, vp, vp, vp, i64, vp, i64, i64, vp, ctypes.c_int, vp, vp, i64, vp, vp,
                                                      ctypes.c_int]),
        "acb_streams_replace_host": (ctypes.c_int, [vp, vp, vp, vp, i64, vp, i64, i64, vp, ctypes.c_int, ctypes.c_int, vp, vp, i64,
                                                    pi64]),
        "acb_last_stream_leftmost_ms": (ctypes.c_int, [ctypes.POINTER(ctypes.c_float), i32]),
        "acb_word_filter_device": (ctypes.c_int, [vp, vp, i64, vp, i64, i64, vp, i64, vp, i64, vp, i64, vp, vp]),
        "acb_scan_host_words": (ctypes.c_int, [vp, vp, i64, vp, i64, i64, vp, i64, vp, i64, pi64, ctypes.c_int, ctypes.c_int]),
        "acb_scan_host_leftmost_words": (ctypes.c_int, [vp, vp, i64, vp, i64, i64, vp, i64, vp, i64, pi64, ctypes.c_int]),
        "acb_replace_host_words": (ctypes.c_int, [vp, vp, vp, i64, vp, i64, i64, vp, i64, ctypes.c_int, vp, vp, i64, pi64]),
        "acb_last_words_ms": (ctypes.c_int, [ctypes.POINTER(ctypes.c_float)]),
        "acb_streams_new_words": (ctypes.c_int, [vp, i64, ctypes.c_int, vp, i64, ctypes.POINTER(vp)]),
        "acb_streams_feed_words_device": (ctypes.c_int, [vp, vp, vp, i64, vp, i64, i64, vp, ctypes.c_int, vp, i64, vp, vp,
                                                         ctypes.c_int]),
        "acb_streams_feed_words_host": (ctypes.c_int, [vp, vp, vp, i64, vp, i64, i64, vp, ctypes.c_int, vp, i64, pi64,
                                                       ctypes.c_int]),
        "acb_table_upload_folded": (ctypes.c_int, [vp, ctypes.c_int, vp, vp, i64, ctypes.POINTER(vp)]),
        "acb_table_upload_folded_map": (ctypes.c_int, [vp, ctypes.c_int, vp, vp, i64, vp, vp, i64, ctypes.POINTER(vp)]),
        "acb_expand_aliases_device": (ctypes.c_int, [vp, vp, i64, vp, i64, vp, vp]),
        "acb_last_fold_ms": (ctypes.c_int, [ctypes.POINTER(ctypes.c_float), i32]),
        "acb_streams_new_folded": (ctypes.c_int, [vp, i64, ctypes.c_int, ctypes.c_int, vp, i64, ctypes.POINTER(vp)]),
        "acb_utf8_work_bytes": (ctypes.c_int, [i64, i64, pi64]),
        "acb_utf8_decode_device": (ctypes.c_int, [ctypes.c_int, vp, i64, vp, i64, i64, ctypes.c_int, vp, i64, vp, vp]),
        "acb_utf8_write_device": (ctypes.c_int, [ctypes.c_int, vp, i64, vp, i64, i64, vp, i64, ctypes.c_int, vp, vp, vp]),
        "acb_utf8_encode_device": (ctypes.c_int, [ctypes.c_int, vp, i64, vp, i64, ctypes.c_int, vp, i64, vp, i64, vp, vp, vp]),
        "acb_last_utf8_ms": (ctypes.c_int, [ctypes.POINTER(ctypes.c_float), i32]),
        "acb_utf8_carry_new": (ctypes.c_int, [ctypes.c_int, i64, ctypes.POINTER(vp)]),
        "acb_utf8_carry_free": (None, [vp]),
        "acb_utf8_carry_reset": (ctypes.c_int, [vp, vp, i64]),
        "acb_utf8_carry_pending": (ctypes.c_int, [vp, vp, i64]),
        "acb_utf8_carry_bytes": (ctypes.c_int, [vp, i32, vp, ctypes.POINTER(ctypes.c_int32)]),
        "acb_utf8_carry_stage_device": (ctypes.c_int, [vp, vp, i64, vp, i64, i64, vp, ctypes.c_int, vp, i64, vp, vp]),
        "acb_utf8_carry_commit_device": (ctypes.c_int, [vp, vp, i64, vp]),
        "acb_launch_count": (i64, []),
        "acb_set_kernel_timing": (ctypes.c_int, [ctypes.c_int]),
        "acb_last_kernel_ms": (ctypes.c_float, []),
        "acb_last_error": (ctypes.c_char_p, []),
        "acb_abi_version": (ctypes.c_int, []),
    }
    for name, (res, args) in sig.items():
        fn = getattr(L, name)
        fn.restype = res
        fn.argtypes = args
    if L.acb_abi_version() != ABI_VERSION:
        raise ImportError(f"{LIB_PATH} has ABI version {L.acb_abi_version()}, this package needs {ABI_VERSION}: "
                          "rebuild it with `python -m pyahocorasick_b200.build --force`")
    _lib = L
    return L


EXPORTED_SYMBOLS = [
    "acb_trie_new", "acb_trie_free", "acb_trie_clear", "acb_trie_add_word", "acb_trie_remove_word",
    "acb_trie_find", "acb_trie_longest_prefix", "acb_trie_make_automaton", "acb_trie_kind",
    "acb_trie_count", "acb_trie_longest_word", "acb_trie_nodes", "acb_trie_links", "acb_trie_host_bytes", "acb_trie_key_order", "acb_trie_key_ranges", "acb_trie_flat_view",
    "acb_trie_content_hash", "acb_trie_flat_save", "acb_trie_flat_load",
    "acb_trie_export_nodes", "acb_trie_import_nodes", "acb_node_records_span",
    "acb_device_count", "acb_table_upload", "acb_table_free", "acb_table_device_bytes",
    "acb_scan_geometry", "acb_table_set_cta_limit", "acb_table_scan_grid",
    "acb_scan_device", "acb_scan_host", "acb_copy_records", "acb_take_records", "acb_release_records", "acb_sort_matches_device", "acb_table_set_long_state", "acb_table_get_long_state",
    "acb_streams_new", "acb_streams_free", "acb_streams_reset", "acb_streams_feed_device", "acb_streams_feed_host",
    "acb_streams_positions", "acb_space_letters", "acb_scan_device_skip", "acb_scan_host_skip", "acb_streams_new_skip",
    "acb_last_skip_ms", "acb_lookup_device", "acb_lookup_host", "acb_table_upload_key_ranges", "acb_select_device",
    "acb_select_host", "acb_leftmost_longest_device", "acb_scan_host_leftmost", "acb_last_leftmost_ms",
    "acb_replacer_new", "acb_replacer_free", "acb_replace_device", "acb_replace_host", "acb_last_replace_ms",
    "acb_streams_new_leftmost", "acb_streams_feed_leftmost_device", "acb_streams_feed_leftmost_host", "acb_streams_replace_device",
    "acb_streams_replace_host", "acb_last_stream_leftmost_ms", "acb_word_filter_device", "acb_scan_host_words",
    "acb_scan_host_leftmost_words", "acb_replace_host_words", "acb_last_words_ms", "acb_streams_new_words",
    "acb_streams_feed_words_device", "acb_streams_feed_words_host", "acb_leftmost_first_device", "acb_scan_host_leftmost_kind",
    "acb_replacer_new_kind", "acb_streams_new_leftmost_kind", "acb_table_upload_folded", "acb_expand_aliases_device",
    "acb_last_fold_ms", "acb_table_upload_folded_map", "acb_streams_new_folded", "acb_utf8_work_bytes", "acb_utf8_decode_device",
    "acb_utf8_write_device", "acb_utf8_encode_device", "acb_last_utf8_ms", "acb_utf8_carry_new",
    "acb_utf8_carry_free", "acb_utf8_carry_reset", "acb_utf8_carry_pending", "acb_utf8_carry_bytes",
    "acb_utf8_carry_stage_device", "acb_utf8_carry_commit_device", "acb_launch_count", "acb_set_kernel_timing",
    "acb_last_kernel_ms", "acb_last_error", "acb_abi_version",
]


def last_error() -> str:
    return (lib().acb_last_error() or b"").decode("utf-8", "replace")


def check(rc: int) -> None:
    """Map a status code to the exception the reference would raise."""
    if rc == ACB_OK:
        return
    msg = last_error()
    if rc == ACB_ENOMEM:
        raise MemoryError(msg)
    if rc == ACB_EINVAL:
        raise ValueError(msg)
    if rc == ACB_ESTATE:
        raise AttributeError(msg)
    if rc == ACB_ERANGE:
        raise OverflowError(msg)
    raise NativeError(f"[{rc}] {msg}")


def ptr(a: np.ndarray) -> ctypes.c_void_p:
    return ctypes.c_void_p(a.ctypes.data)
