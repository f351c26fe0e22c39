/*
 * acb200.h -- C ABI of the H100-native Aho-Corasick batch-search path.
 *
 * This is the drop-in boundary: plain pointers and sizes, no torch / Python types.
 * The reference (WojciechMula/pyahocorasick v2.2.0) has no C plugin ABI of its own --
 * the path sits behind the CPython type `ahocorasick.Automaton`
 * (src/Automaton.c:1204-1230 method table, src/pyahocorasick.c:67-137 module init).
 * Each entry point below names the reference function whose role it takes over; the
 * Python class pyahocorasick_b200.Automaton (ctypes) keeps the reference's signatures
 * and exceptions on top of these calls.  INTEGRATION.md shows the binding a
 * maintainer of the reference would add.
 *
 * Conventions
 *   - every function that can fail returns an int status: ACB_OK (0) or a negative
 *     ACB_E* code; acb_last_error() returns a thread-local human-readable message.
 *   - keys and haystacks are BYTE strings.  Wider letters (the reference's unicode
 *     flavour, KEY_SEQUENCE) are passed as little-endian fixed-width letters with
 *     `letter_bytes` in {1,2,4}; matches are only reported at letter boundaries and
 *     end_index is counted in letters, exactly like the reference's index into
 *     its TRIE_LETTER_TYPE array (src/common.h:51-67).
 *   - the library never falls back to a CPU search: acb_scan_* fail with
 *     ACB_ECUDA when no device / kernel image is available.
 */
#ifndef ACB200_H_INCLUDED
#define ACB200_H_INCLUDED

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ACB_ABI_VERSION 5

enum {
    ACB_OK        =  0,
    ACB_ENOMEM    = -1,   /* -> MemoryError   (reference: PyErr_NoMemory everywhere)           */
    ACB_EINVAL    = -2,   /* -> ValueError / TypeError at the Python layer                      */
    ACB_ESTATE    = -3,   /* automaton not in the AHOCORASICK state (src/Automaton.c:886-891)   */
    ACB_ECUDA     = -4,   /* CUDA runtime / launch failure, no device, no sm_90a image           */
    ACB_EOVERFLOW = -5,   /* match buffer too small: *n_found holds the required capacity        */
    ACB_ERANGE    = -6    /* size beyond what int32 state ids / end_index can hold               */
};

/* same numeric values as the reference's AutomatonKind (src/Automaton.h:16-20) */
enum { ACB_EMPTY = 0, ACB_TRIE = 1, ACB_AHOCORASICK = 2 };

/* One reported occurrence.  The Python layer maps key_id -> value so that
 * (end_index, value) equals what src/AutomatonSearchIter.c:178-190 builds. */
typedef struct acb_match {
    int32_t hay_id;      /* index of the haystack inside the batch            */
    int32_t end_index;   /* index of the LAST letter of the occurrence        */
    int32_t key_id;      /* caller-chosen id given to acb_trie_add_word       */
} acb_match;

/* ------------------------------------------------------------------ host --- */

/* Host-side trie + automaton.  Replaces the TrieNode/Pair heap graph
 * (src/trienode.h:19-42) with an arena of int32 node ids. */
typedef struct acb_trie acb_trie;

acb_trie *acb_trie_new(int letter_bytes);                 /* automaton_new, src/Automaton.c:96-181 */
void      acb_trie_free(acb_trie *t);
int       acb_trie_clear(acb_trie *t);                    /* automaton_clear                       */

/* trie_add_word (src/trie.c:14-63) + value slot of automaton_add_word
 * (src/Automaton.c:201-300).  key_id >= 0 is stored on the terminal node.
 * *prev_key_id receives the id previously stored there, or -1 for a new key.
 * nbytes must be a positive multiple of letter_bytes; nbytes == 0 is a no-op that
 * sets *prev_key_id = -2 (the reference returns False for an empty key, :257). */
int acb_trie_add_word(acb_trie *t, const uint8_t *key, int64_t nbytes, int32_t key_id,
                      int32_t *prev_key_id);

/* trie_remove_word (src/trie.c:66-136): *key_id = removed id or -1 if absent. */
int acb_trie_remove_word(acb_trie *t, const uint8_t *key, int64_t nbytes, int32_t *key_id);

/* trie_find / automaton_exists / automaton_match (src/trie.c:139-155):
 * *key_id = id of the key equal to `key` (or -1); *is_prefix = 1 when `key` is a
 * prefix of at least one live key. */
int acb_trie_find(const acb_trie *t, const uint8_t *key, int64_t nbytes, int32_t *key_id,
                  int32_t *is_prefix);

/* trie_longest (src/trie.c:158-174): number of leading LETTERS of `key` that
 * follow existing edges. */
int64_t acb_trie_longest_prefix(const acb_trie *t, const uint8_t *key, int64_t nbytes);

/* automaton_make_automaton (src/Automaton.c:560-649): BFS failure links, then --
 * new in this build -- flatten to the int32 tables the device scans.
 * Returns ACB_OK; *built = 1 when the state went TRIE -> AHOCORASICK, 0 when there
 * was nothing to do (the reference returns False, :574-575). */
int acb_trie_make_automaton(acb_trie *t, int32_t *built);

int     acb_trie_kind(const acb_trie *t);          /* ACB_EMPTY / ACB_TRIE / ACB_AHOCORASICK */
int64_t acb_trie_count(const acb_trie *t);         /* live keys   (len(A))                   */
int64_t acb_trie_longest_word(const acb_trie *t);  /* in letters  (Automaton.longest_word)   */
int64_t acb_trie_nodes(const acb_trie *t);         /* live nodes  (get_stats nodes_count)    */
int64_t acb_trie_links(const acb_trie *t);         /* live edges  (get_stats links_count)    */
int64_t acb_trie_host_bytes(const acb_trie *t);    /* bytes of the node arena + edge table (get_stats total_size) */

/* The ids of the live keys in the order in which the reference's keys() / values() / items() yield them: a pre-order
 * walk that takes a node's most recently linked child first (its iterator pushes the children in array order and pops
 * the last, src/AutomatonItemsIter.c:125-288).  *n = number of live keys; ACB_EOVERFLOW when cap is smaller. */
int acb_trie_key_order(const acb_trie *t, int32_t *out, int64_t cap, int64_t *n);

/* Read-only view of the flattened automaton (valid until the trie changes).
 * State ids are BFS order, root = 0.  Used for upload and for white-box tests. */
typedef struct acb_flat_view {
    int32_t        n_states;      /* S                                                        */
    int32_t        n_classes;     /* K; class 0 = "byte that occurs in no key"                */
    int32_t        n_keys;        /* 1 + largest key_id                                       */
    int32_t        letter_bytes;
    int32_t        min_key_bytes; /* shortest live key                                        */
    int32_t        max_key_bytes;
    const uint8_t *byte_class;    /* [256]  byte -> class                                     */
    const int32_t *goto_cm;       /* [K*S]  column-major: goto_cm[c*S+s] = child or -1        */
    const int32_t *fail;          /* [S]    failure link, fail[0] = -1 (root has none, A12)   */
    const int32_t *letter_fail;   /* [S]    fail link between letter-aligned states (== fail for 1-byte letters), root -1 */
    const int32_t *key_of;        /* [S]    key_id ending exactly at this state, or -1        */
    const int32_t *out_ptr;       /* [S+1]  CSR over out_idx                                  */
    const int32_t *out_idx;       /* key ids on the chain s, fail(s), ... (longest first)     */
    const int32_t *key_len;       /* [n_keys] key length in LETTERS (0 = unused id)           */
    /* prefilter (see DESIGN.md "filter kernel") */
    int32_t        gram_bytes;    /* g : bytes hashed per probe                               */
    int32_t        stride;        /* s : probe every s-th byte position                       */
    int32_t        log2_bits1;    /* n: the gram bitmap has 2^n bits (shared memory on the device), 2^(n-5) words */
    int32_t        log2_anchor_slots; /* anchor table has 2^n slots of 8 uint32 (32 B)        */
    int32_t        log2_bits3;    /* tag bitmap (global memory) has 2^k bits; 0 = not built    */
    const uint32_t *bitmap1;      /* single placement: a gram sets two bits of one word, word = umulhi(hash1, 2^(n-5));
                                     pair placement: acb_pair_place / acb_pair_place2 (csrc/acb_hash.h), 2^(n-5) + 2^(k-5) words */
    const uint32_t *bitmap3;      /* 1<<(k-5) words: bit = (hash2|1) * 0x9E3779B1 >> (32-k); only for key sets the shared-memory filter cannot hold */
    const uint32_t *anchors;      /* slot: tag(hash2|1, 0=empty), key_id(-1=MULTI), j|len<<8|last<<16, 20 bytes */
    int32_t        filter_flags;  /* ACB_FILTER_* : how the bitmap places a gram (csrc/acb_hash.h) */
    int32_t        log2_bits2;    /* PAIR placement: level 2 (2^k bits, keyed by the anchor tag) follows level 1 in bitmap1; else 0 */
} acb_flat_view;

/* filter_flags */
#define ACB_FILTER_WIDE 1   /* single placement, g % 4 == 0: the first bit comes from the high half of the 64-bit hash sum */
#define ACB_FILTER_PAIR 2   /* pair placement (gram 4, stride 1, 1-byte letters): two adjacent positions share one word,
                               one bit per (role, remaining byte); level 2 keyed by the anchor tag behind it                */

int acb_trie_flat_view(const acb_trie *t, acb_flat_view *out);

/* ---- the flat-table cache (SURVEY.md section 8(f) #2, last clause) ---------------------------------------
 * A loaded or unpickled automaton of kind AHOCORASICK is searchable at once in the reference, whose files carry the
 * failure links (src/custompickle/load/module_automaton_load.c:85-93, src/Automaton.c:139-145).  Here the links are a
 * function of the key set, so what is cached is everything make_automaton derives from it: acb_trie_flat_save writes
 * the flattened tables (goto / fail / outputs / filter / anchors) with a content hash of the key set as
 * make_automaton numbers it; acb_trie_flat_load installs them on a trie that holds the same keys (kind TRIE) and turns
 * it into an automaton without the BFS, the flatten and the filter construction.  ACB_EINVAL when the blob does not
 * belong to this key set or library version: call acb_trie_make_automaton then.
 * acb_trie_flat_save: call with out == NULL first, *need is always set. */
uint64_t acb_trie_content_hash(const acb_trie *t);
int acb_trie_flat_save(const acb_trie *t, uint8_t *out, int64_t cap, int64_t *need);
int acb_trie_flat_load(acb_trie *t, const uint8_t *buf, int64_t len);

/* ---- the reference's on-disk node records (SURVEY.md section 8(f) #2) -------------------------------
 * Both of the reference's serialisations write one record per trie node, in pre-order (`trie_traverse`,
 * src/trie.c:196-225), children in table order:
 *     { u64 output; u64 fail; u32 n; u8 eow; 3 pad }  =  PICKLE_TRIENODE_SIZE, src/pickle/pickle.h:7
 *     n x { letter (2 bytes in the bytes build, 4 in the unicode build); u64 child }   (packed `Pair`, src/trienode.h:19-25)
 * `__reduce__` (src/Automaton_pickle.c:128-188) numbers the nodes 1..N and stores those numbers in `fail`/`child`;
 * `save` (src/custompickle/save/automaton_save.c:85-138) stores node addresses instead, each record preceded by its own
 * address, and -- for STORE_ANY -- followed by the serialised value whose size is written into `output`.
 *
 * acb_trie_export_nodes writes the records with ids 1..N (which double as the "addresses" of a save file).
 * Call it with out == NULL first: *need_bytes and *n_nodes are always set.  value_of_key (nullable) supplies
 * `output` of end-of-word nodes (STORE_INTS / STORE_LENGTH); rec_off[N+1] (nullable) receives the byte offset
 * of every record, eow_key[N] (nullable) the key id ending at the node or -1.  `fail` is written only for a
 * built automaton (ACB_AHOCORASICK), else 0.  Letters: letter_width 2 sign-extends 1-byte letters exactly
 * like the bytes build does (src/utils.c:199-202). */
int acb_trie_export_nodes(const acb_trie *t, int letter_width, const int64_t *value_of_key, int64_t n_values,
                          uint8_t *out, int64_t cap, int64_t *need_bytes, int64_t *n_nodes,
                          int64_t *rec_off, int32_t *eow_key, int64_t cap_nodes);

/* The inverse: parse n_nodes records and enter every key into the (empty) trie t, key ids 0.. in pre-order.
 * mode ACB_NODES_PICKLE: records back to back, node i has id i+1 (src/Automaton_pickle.c:330-456);
 * mode ACB_NODES_SAVE: `u64 address` before each record, and `output` bytes of serialised value after each
 * end-of-word record when store_any != 0 (src/custompickle/load/module_automaton_load.c:108-180).
 * out_value[k] = `output` of key k's node, out_blob_off[k] = offset of its serialised value in buf (SAVE + store_any)
 * or -1.  Fail links in the file are ignored: acb_trie_make_automaton recomputes them.
 * Returns ACB_EINVAL for truncated / malformed input (dangling child, node reachable twice, letter out of range). */
enum { ACB_NODES_PICKLE = 0, ACB_NODES_SAVE = 1 };
int acb_trie_import_nodes(acb_trie *t, const uint8_t *buf, int64_t len, int64_t n_nodes, int letter_width, int mode,
                          int store_any, int64_t *out_value, int64_t *out_blob_off, int64_t cap_keys, int64_t *n_keys,
                          int64_t *consumed,
                          uint8_t *key_bytes, int64_t key_cap, int64_t *key_off /* cap_keys + 1 */, int64_t *key_need);
/* key_bytes / key_off (nullable) receive the keys themselves, key k = key_bytes[key_off[k] .. key_off[k+1]);
 * *key_need (nullable) is always set to the total.  Sizes are not known in advance: import into a scratch trie
 * first (all outputs NULL except n_keys / key_need), then for real. */

/* bytes taken by n_nodes back-to-back records (the used part of one pickle chunk, src/Automaton_pickle.c:362-419) */
int acb_node_records_span(const uint8_t *buf, int64_t len, int64_t n_nodes, int letter_width, int64_t *span);

/* ---------------------------------------------------------------- device --- */

/* The flattened automaton resident in HBM of one GPU (uploaded once). */
typedef struct acb_table acb_table;

int  acb_device_count(int32_t *n);
int  acb_table_upload(const acb_trie *t, int device, acb_table **out);
void acb_table_free(acb_table *tb);
int64_t acb_table_device_bytes(const acb_table *tb);

/* which scan kernel to run */
enum {
    ACB_ALGO_AUTO   = 0,
    ACB_ALGO_FILTER = 1,  /* gram-filter + trie walk (start-anchored), the fast path          */
    ACB_ALGO_DFA    = 2,  /* goto/fail automaton walk with CSR outputs, one lane per chunk     */
    ACB_ALGO_LONG   = 3   /* iter_long semantics (src/AutomatonSearchIterLong.c:89-153): longest,
                             non-overlapping matches; one lane per haystack                       */
};

/* Batch scan, DEVICE buffers, asynchronous on `stream` (a cudaStream_t / CUstream).
 * Replaces the loop in automaton_search_iter_next (src/AutomatonSearchIter.c:243-300)
 * and automaton_find_all (src/Automaton.c:693-714) for a whole batch at once.
 *
 *   d_hay      : all haystacks back to back, total_bytes bytes
 *   d_offsets  : n_hay+1 byte offsets (int64, multiples of letter_bytes), or NULL
 *                when every haystack is `stride_bytes` long (haystack h = [h*stride, (h+1)*stride))
 *   d_out/cap  : match records; records beyond cap are counted but not stored
 *   d_count    : device int64; incremented by the number of matches found
 *                (the caller zeroes it; order of records is unspecified).
 * One scan at a time per table: the table owns the scratch buffers of the scan.
 */
int acb_scan_device(acb_table *tb, const uint8_t *d_hay, int64_t total_bytes,
                    const int64_t *d_offsets, int64_t n_hay, int64_t stride_bytes,
                    acb_match *d_out, int64_t cap, int64_t *d_count,
                    void *stream, int algo);

/* Batch scan, HOST buffers: H2D copy of haystacks (+offsets), the kernel, and D2H of
 * the count and the records, all inside the call (this is what `e2e` times).
 * Returns ACB_EOVERFLOW (and the needed size in *n_found) when cap is too small.
 * If sort != 0 the records come back in the reference's order:
 * hay_id, then end_index ascending, then longest key first (SURVEY 3.3).
 * `out` may be NULL (then `cap` only bounds the device buffer): the records stay in the
 * table's pinned staging area and acb_copy_records() copies them out once the count is known. */
int acb_scan_host(acb_table *tb, const uint8_t *hay, int64_t total_bytes,
                  const int64_t *offsets, int64_t n_hay, int64_t stride_bytes,
                  acb_match *out, int64_t cap, int64_t *n_found, int algo, int sort);

/* copy the first n records of the last acb_scan_host(out = NULL) call into `out` */
int acb_copy_records(acb_table *tb, acb_match *out, int64_t n);

/* ... or take them without a copy: *ptr is the pinned staging buffer itself (*n records, room for *cap), owned
 * by the caller from now on and to be given back with acb_release_records(ptr, cap) when done -- it then serves a
 * later scan.  *ptr == NULL when the last scan found nothing. */
int  acb_take_records(acb_table *tb, acb_match **ptr, int64_t *n, int64_t *cap);
void acb_release_records(acb_match *ptr, int64_t cap);

/* Sort n device-resident records into the reference's order (hay_id, end_index ascending, longest
 * key first) with a 64-bit radix sort, asynchronously on `stream`.  max_hay_letters bounds end_index.
 * ACB_ERANGE when hay_id/end_index/length do not fit one 64-bit key (sort on the host then). */
int acb_sort_matches_device(acb_table *tb, acb_match *d_records, int64_t n, int64_t n_hay,
                            int64_t max_hay_letters, void *stream);

/* iter_long streaming (src/AutomatonSearchIterLong.c:156-212: set() keeps iter->state): the walk state carried from one
 * chunk to the next stays a state id, nothing of the old text is scanned again.
 * acb_table_set_long_state: the state (BFS id, 0 = root) in which haystack 0 of the NEXT ACB_ALGO_LONG scan starts; one
 *   shot, every other haystack and every later scan start at the root.  ACB_EINVAL for an id that is not a state.
 * acb_table_get_long_state: the state in which haystack 0 of the LAST ACB_ALGO_LONG scan ended (its text exhausted,
 *   a match still pending at the end reported: then the root).  After acb_scan_device the caller synchronises its
 *   stream first. */
int acb_table_set_long_state(acb_table *tb, int32_t state);
int acb_table_get_long_state(acb_table *tb, int32_t *state);

/* number of kernel launches issued by this library so far (bench.py's gpu_launches) */
int64_t acb_launch_count(void);

/* timing of the most recent scan kernel on its own stream, in milliseconds, measured
 * with CUDA events recorded around the launch (0 when timing is disabled). */
int   acb_set_kernel_timing(int enabled);
float acb_last_kernel_ms(void);

const char *acb_last_error(void);
int         acb_abi_version(void);

#ifdef __cplusplus
}
#endif
#endif /* ACB200_H_INCLUDED */
