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
 *   - an entry point that runs on the device of its table, stream batch or replacer
 *     leaves the calling thread's current CUDA device as it found it, on every
 *     return path, errors included.
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

/* That order as ranges over the flattened automaton (acb_trie_flat_view; ACB_ESTATE before it is built).  In a pre-order
 * walk the keys at or under a node are one run, so for every state s that ends a whole letter (every state for 1-byte
 * letters): the run is order[lo[s] .. lo[s] + cnt[s]) -- the node's own key first, if it ends one -- and its
 * letter-children are child[child_ptr[s] .. child_ptr[s+1]), youngest first, which is by ascending lo.  States inside a
 * letter have cnt 0 and no children.  Sizes: order acb_trie_count(t); lo, cnt n_states; child_ptr n_states + 1; child
 * n_states (always enough); *n_edges = the entries of child used. */
int acb_trie_key_ranges(const acb_trie *t, int32_t *order, int32_t *lo, int32_t *cnt, int32_t *child_ptr, int32_t *child,
                        int64_t *n_edges);

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

/* Test hooks: the scan kernels' tile rings, and launches on fewer SMs, so that a test can make one CTA go round its
 * ring many times on a short text.
 * acb_scan_geometry: the ring of acb_pair_kernel (pair != 0) or of acb_stream_kernel, from the constants the kernels
 *   are compiled with: out[0..5] = slice bytes, tile bytes, stages, consumer warps, tile claims in flight per CTA,
 *   look-ahead bytes copied past a tile.  n is the room in out (at least 6).  Needs no device.
 * acb_table_set_cta_limit: n = 0 (the default) launches as the device allows, one persistent scan CTA per SM; n > 0
 *   launches as if the device had min(n, SMs) SMs: the grid of the persistent scan kernels and the bound of the
 *   grid-stride loops (a few blocks per SM) shrink, allocations sized by the SM count stay.  Results are the same.
 * acb_table_scan_grid: the launch of a filter scan of one segment of total_bytes (at most 2 GiB) under the current
 *   limit: its CTAs and the tiles they claim.  The scans compute their launch shape with this very function. */
int acb_scan_geometry(int pair, int32_t *out, int32_t n);
int acb_table_set_cta_limit(acb_table *tb, int32_t n);
int acb_table_scan_grid(const acb_table *tb, int64_t total_bytes, int32_t *grid, int64_t *n_tiles);

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
 *   d_hay      : all haystacks back to back, total_bytes bytes; 16-byte aligned (the scan reads it with TMA bulk
 *                copies), else ACB_EINVAL.  A view into a larger buffer that starts elsewhere must be copied first.
 *   d_offsets : n_hay+1 byte offsets (int64, multiples of letter_bytes), or NULL
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
 *   stream first.
 * An ACB_ALGO_LONG scan without text (total_bytes == 0 or n_hay == 0) or without keys consumes the state set before it
 *   like any other: haystack 0 ends where it started, so acb_table_get_long_state returns that state, and the next
 *   scan starts at the root. */
int acb_table_set_long_state(acb_table *tb, int32_t state);
int acb_table_get_long_state(acb_table *tb, int32_t *state);

/* ---- stream batches: the next chunk of many streams in one call ---------------------------------------------------
 * The batch form of iter().set() / iter_long().set() (src/AutomatonSearchIter.c:303-368,
 * src/AutomatonSearchIterLong.c:156-212).  An acb_streams holds, in HBM, what every stream carries from one chunk to
 * the next: the letters consumed so far, and either its last longest_word - 1 letters (find_all semantics: a feed
 * reports every match that ends inside the chunk, including those that start in earlier chunks) or the iter_long walk
 * state (long_mode != 0: a feed continues each stream's longest-match walk).
 *
 * The table is passed to every call and not kept: acb_streams remembers the device, letter width, tail length and
 * (long mode) state count of the table it was made for and refuses another (ACB_EINVAL).
 *
 * A feed takes chunks in the forms of acb_scan_device / acb_scan_host; ids[h] (int32, distinct, in [0, n_streams))
 * names the stream chunk h continues, ids == NULL means chunk h continues stream h (then n_chunks <= n_streams).
 * Streams without a chunk do not move.  Records: hay_id = index of the chunk in the call, end_index = letter of the
 * chunk (add the stream's position before the feed, see acb_streams_positions, for the position in the stream).
 * Overflow commits nothing: a host feed that returns ACB_EOVERFLOW, or a device feed that leaves *d_count > cap,
 * changes no stream, and the same feed can be repeated with a larger buffer.
 * Feeds of one stream batch must not overlap in time: issue them on one CUDA stream (or synchronise in between). */
typedef struct acb_streams acb_streams;

int  acb_streams_new(const acb_table *tb, int64_t n_streams, int long_mode, acb_streams **out);
void acb_streams_free(acb_streams *ss);

/* stream ids[0..n) (ids == NULL: every stream) back to position 0 with nothing carried (set(x, reset=True)).
 * Synchronises the device. */
int acb_streams_reset(acb_streams *ss, const int32_t *ids, int64_t n);

/* DEVICE buffers, asynchronous on `stream`.  Zeroes *d_count itself, then counts every record (stored up to cap).
 * d_chunks must be 16-byte aligned, as d_hay of acb_scan_device, else ACB_EINVAL.  d_ids is not checked: the caller guarantees distinct ids in range.  algo: ACB_ALGO_AUTO, _FILTER or _DFA for a
 * find_all batch (the scan of the chunks; seams are always walked), ACB_ALGO_AUTO or _LONG for an iter_long batch.
 * Records are unsorted: acb_sort_matches_device(tb, d_out, n, n_chunks, longest chunk in letters, stream). */
int acb_streams_feed_device(acb_streams *ss, acb_table *tb, const uint8_t *d_chunks, int64_t total_bytes,
                            const int64_t *d_offsets, int64_t n_chunks, int64_t stride_bytes, const int32_t *d_ids,
                            acb_match *d_out, int64_t cap, int64_t *d_count, void *stream, int algo);

/* HOST buffers, like acb_scan_host (out may be NULL: acb_copy_records / acb_take_records on tb).  ids are checked:
 * ACB_EINVAL for a duplicate or an id out of range, before anything runs. */
int acb_streams_feed_host(acb_streams *ss, acb_table *tb, const uint8_t *chunks, int64_t total_bytes,
                          const int64_t *offsets, int64_t n_chunks, int64_t stride_bytes, const int32_t *ids,
                          acb_match *out, int64_t cap, int64_t *n_found, int algo, int sort);

/* letters consumed by every stream since its start or its last reset (cap >= n_streams).  Synchronises the device. */
int acb_streams_positions(acb_streams *ss, int64_t *out, int64_t cap);

/* ---- white space: iter(..., ignore_white_space=1) for a whole batch (src/AutomatonSearchIter.c:270-274) ------------
 * A skip set is a sorted array of distinct letter values, exactly as the letters are stored in the buffer (1-, 2- or
 * 4-byte little-endian values of the table's width; a unicode-flavour latin-1 table has 1-byte letters), at most
 * ACB_MAX_SKIP long.  The skip scans behave as if every letter of the set were removed from each haystack before the
 * scan, and report end_index in letters of the ORIGINAL haystack: the batch is compacted on the device, scanned by
 * the ordinary kernels, and each stored record is mapped back.  ACB_EINVAL for ACB_ALGO_LONG (iter_long has no such
 * option), an unsorted or too large set.  Records beyond cap are counted exactly, as by the plain scans. */
#define ACB_MAX_SKIP 1024

/* Every letter of the given width for which libc iswspace() is true under the current LC_CTYPE, in ascending order:
 * letter_bytes 1 (with signed_bytes != 0 the predicate sees the byte widened through a signed char, as the reference's
 * bytes build does; out receives the byte values), 2 (all 65 536 values) or 4 (0 .. 0x10FFFF).  *n is always set;
 * ACB_EOVERFLOW when cap is smaller.  Host only, no device needed. */
int acb_space_letters(int letter_bytes, int signed_bytes, uint32_t *out, int64_t cap, int64_t *n);

/* acb_scan_device with a skip set (host array).  Zeroes *d_count itself.  Asynchronous on `stream` except that it
 * waits once for the compaction, to learn the compacted size the scan kernels are launched for.  d_out holds the
 * records in ORIGINAL coordinates once the stream reaches them.  The compacted batch and the map back live in a
 * workspace of the table, reused by every skip call and skip feed on it: the next such call, on any CUDA stream, first
 * waits (cudaStreamWaitEvent) for the work of this one that still reads it.  As for acb_scan_device, one scan at a time
 * per table. */
int acb_scan_device_skip(acb_table *tb, const uint8_t *d_hay, int64_t total_bytes,
                         const int64_t *d_offsets, int64_t n_hay, int64_t stride_bytes,
                         acb_match *d_out, int64_t cap, int64_t *d_count, void *stream, int algo,
                         const uint32_t *skip, int64_t n_skip);

/* acb_scan_host with a skip set: upload, compact, scan, map back, sort, copy back in one call (no pipeline).
 * out == NULL works as for acb_scan_host (acb_copy_records / acb_take_records). */
int acb_scan_host_skip(acb_table *tb, const uint8_t *hay, int64_t total_bytes,
                       const int64_t *offsets, int64_t n_hay, int64_t stride_bytes,
                       acb_match *out, int64_t cap, int64_t *n_found, int algo, int sort,
                       const uint32_t *skip, int64_t n_skip);

/* A find_all stream batch whose feeds skip the letters of `skip` (copied): stream s reports what iter(c0,
 * ignore_white_space=1) ... .set(c1) ... reports.  Positions (acb_streams_positions, end_index) count ORIGINAL letters;
 * the tail carried to the next chunk holds the last T kept letters, so a key that white space splits across a chunk
 * boundary is found.  acb_streams_feed_*, _reset and _positions serve it unchanged. */
int acb_streams_new_skip(const acb_table *tb, int64_t n_streams, const uint32_t *skip, int64_t n_skip, acb_streams **out);

/* With kernel timing on (acb_set_kernel_timing), the milliseconds of the compaction kernel and of the map-back kernel
 * of the last skip scan or skip feed on this thread, from CUDA events around each launch (the call then waits for
 * them); 0 when timing is off or the call launched none.  acb_last_kernel_ms() gives its scan kernel. */
int acb_last_skip_ms(float *compact_ms, float *remap_ms);

/* ---- dictionary lookups: exists / match / longest_prefix / get for many keys at once -------------------------------
 * trie_find / trie_longest (src/trie.c:139-174) for n_keys queries at once.  key_id[i]: id of the key equal to query i
 * or -1 (always -1 for an empty query); prefix[i]: leading LETTERS of query i that follow trie edges (a letter walked
 * only in part does not count), so query i is a prefix of some key exactly when prefix[i] equals its length in letters.
 * prefix never exceeds the longest key.  Queries as acb_scan_device's haystacks (d_offsets: n_keys+1 int64 byte
 * offsets, multiples of letter_bytes, or NULL and stride_bytes >= 0 for keys of one length); unlike the scans, the
 * keys need no alignment.  One lane per query walks the goto table of the uploaded automaton from the root.
 *
 * DEVICE buffers, asynchronous on `stream`.  d_offsets is not checked.  With kernel timing on (acb_set_kernel_timing)
 * the call waits for its kernel and acb_last_kernel_ms() gives its time. */
int acb_lookup_device(acb_table *tb, const uint8_t *d_keys, int64_t total_bytes, const int64_t *d_offsets,
                      int64_t n_keys, int64_t stride_bytes, int32_t *d_key_id, int32_t *d_prefix, void *stream);

/* HOST buffers: upload, kernel, copy back, synchronous.  The offsets are checked (ACB_EINVAL) before anything runs.
 * The scratch buffers belong to the table: one call at a time per table, as for the scans.  Without a device:
 * ACB_ECUDA (there is no CPU fallback). */
int acb_lookup_host(acb_table *tb, const uint8_t *keys, int64_t total_bytes, const int64_t *offsets,
                    int64_t n_keys, int64_t stride_bytes, int32_t *key_id, int32_t *prefix);

/* ---- dictionary selection: keys / values / items (prefix, wildcard, how) for many patterns at once ------------------
 * The ranges of acb_trie_key_ranges go to the device once, before the first select call: t is the trie the table was
 * uploaded from, unchanged since.  A repeated call returns at once; the table frees them.  About 12 bytes per state plus
 * 4 per key and per letter edge.  The scans and lookups do not need them. */
int acb_table_upload_key_ranges(acb_table *tb, const acb_trie *t);

/* how, as the reference's MATCH_* constants (src/AutomatonItemsIter.h) */
#define ACB_MATCH_EXACT_LENGTH     0
#define ACB_MATCH_AT_MOST_PREFIX   1
#define ACB_MATCH_AT_LEAST_PREFIX  2

/* keys(pattern, wildcard, how) (src/AutomatonItemsIter.c:125-288) for n patterns at once: the ids of pattern i's keys
 * are key_id[out_offsets[i] .. out_offsets[i+1]), in the order acb_trie_key_order gives them.  wildcard: a letter value
 * that matches any letter, or -1 for none; without one, `how` is ignored and the keys are those that start with the
 * pattern (the reference's prefix query).  With one, how = EXACT_LENGTH: keys of the pattern's length that match it
 * letter by letter; AT_MOST_PREFIX: keys that match a prefix of the pattern; AT_LEAST_PREFIX: keys whose prefix matches
 * the pattern.  Patterns are laid out as acb_lookup_device's keys (no alignment needed).  ACB_ESTATE before
 * acb_table_upload_key_ranges.
 *
 * DEVICE buffers, asynchronous on `stream`: d_out_offsets (n+1 int64) and *d_total are always written; d_key_id only
 * when the total is at most cap (the kernel checks it on the device).  Two passes: one counts the keys of every
 * pattern, an exclusive scan gives the offsets, the other writes the ids.  d_offsets is not checked. */
int acb_select_device(acb_table *tb, const uint8_t *d_patterns, int64_t total_bytes, const int64_t *d_offsets, int64_t n,
                      int64_t stride_bytes, int64_t wildcard, int how, int64_t *d_out_offsets, int32_t *d_key_id,
                      int64_t cap, int64_t *d_total, void *stream);

/* HOST buffers, synchronous.  The offsets and the arguments are checked (ACB_EINVAL) before anything runs.  out_offsets
 * and *total are always written; key_id when *total <= cap, else ACB_EOVERFLOW.  Without a device: ACB_ECUDA. */
int acb_select_host(acb_table *tb, const uint8_t *patterns, int64_t total_bytes, const int64_t *offsets, int64_t n,
                    int64_t stride_bytes, int64_t wildcard, int how, int64_t *out_offsets, int32_t *key_id, int64_t cap,
                    int64_t *total);

/* ---- leftmost-longest non-overlapping matches ----------------------------------------------------------------------
 * From the full match list of each haystack (what iter() reports, start = end_index - len + 1): p = 0; while some match
 * starts at or after p, take the smallest such start, the longest match there, and continue at its end_index + 1.  This
 * is not iter_long (src/AutomatonSearchIterLong.c:89-153), whose restart rule depends on the trie's inner nodes.
 *
 * DEVICE buffers, asynchronous on `stream`: d_records holds the full list of n records of a batch of n_hay haystacks,
 * in any order (what acb_scan_device leaves); max_hay_letters bounds end_index.  The chosen records go to d_out in
 * haystack order, then end_index ascending; *d_count is increased by their number and only the first cap are stored.
 * d_records is not changed.  The scratch space belongs to the table: the next call waits (cudaStreamWaitEvent) for the
 * work of this one, also on another CUDA stream.  ACB_ERANGE for more than 2^31-1 records. */
int acb_leftmost_longest_device(acb_table *tb, const acb_match *d_records, int64_t n, int64_t n_hay, int64_t max_hay_letters,
                                acb_match *d_out, int64_t cap, int64_t *d_count, void *stream);

/* HOST buffers: upload, scan (algo ACB_ALGO_AUTO, _FILTER or _DFA; monolithic, as for ACB_ALGO_DFA), select, copy back,
 * synchronous.  *n_found is the exact number of chosen records; ACB_EOVERFLOW when it exceeds cap.  The full list is
 * kept in a device buffer of the table grown to fit.  out == NULL works as for acb_scan_host (acb_copy_records /
 * acb_take_records).  Without a device: ACB_ECUDA. */
int acb_scan_host_leftmost(acb_table *tb, const uint8_t *hay, int64_t total_bytes, const int64_t *offsets, int64_t n_hay,
                           int64_t stride_bytes, acb_match *out, int64_t cap, int64_t *n_found, int algo);

/* ---- leftmost-first: the same rule with priority by key order --------------------------------------------------
 * Among the matches at the smallest start >= p, the one with the smallest key id (the order in which the keys were
 * first added) instead of the longest.  One selection kind says which rule a call follows; the entries below take it
 * where the rule is not in the name.  Every other entry selects leftmost-longest. */
#define ACB_SELECT_LONGEST 0
#define ACB_SELECT_FIRST   1

/* acb_leftmost_longest_device's contract, the leftmost-first rule */
int acb_leftmost_first_device(acb_table *tb, const acb_match *d_records, int64_t n, int64_t n_hay, int64_t max_hay_letters,
                              acb_match *d_out, int64_t cap, int64_t *d_count, void *stream);

/* acb_scan_host_leftmost (n_bits < 0 and bits == NULL: no word set) or acb_scan_host_leftmost_words (a word set as
 * there) under selection kind `kind` (ACB_EINVAL for another value) */
int acb_scan_host_leftmost_kind(acb_table *tb, int kind, const uint8_t *hay, int64_t total_bytes, const int64_t *offsets,
                                int64_t n_hay, int64_t stride_bytes, const uint32_t *bits, int64_t n_bits, acb_match *out,
                                int64_t cap, int64_t *n_found, int algo);

/* With kernel timing on (acb_set_kernel_timing), the milliseconds of the last selection's stages on this thread: sort,
 * candidates, successors, chain, emit (the first n of them, n <= 5), from CUDA events between the stages (the call then
 * waits for them); 0 when timing is off. */
int acb_last_leftmost_ms(float *ms, int32_t n);

/* ---- leftmost-longest replacement ----------------------------------------------------------------------------------
 * Each haystack with the letters [end_index - len + 1, end_index] of every match the leftmost-longest selection chose
 * replaced by that key's replacement, every other letter copied.  A replacer holds the replacement of every key id on
 * the device: rep[rep_offsets[k] .. rep_offsets[k+1]) (bytes, letters of the table's width; ids of removed keys get
 * empty entries).  It records the table's device and letter width and n_ids; the calls refuse (ACB_EINVAL) a table of
 * another device or width, or with more key ids.  The table is passed to every call and not kept, as for stream
 * batches.  The offsets are checked (ACB_EINVAL) before anything runs.  Without a device: ACB_ECUDA. */
typedef struct acb_replacer acb_replacer;

int  acb_replacer_new(const acb_table *tb, const uint8_t *rep, int64_t rep_bytes, const int64_t *rep_offsets, int64_t n_ids,
                      acb_replacer **out);
void acb_replacer_free(acb_replacer *r);

/* A replacer of selection kind `kind`: acb_replace_host, acb_replace_host_words and the replacing stream feeds rewrite
 * the matches that rule chooses.  acb_replacer_new makes one of kind ACB_SELECT_LONGEST. */
int  acb_replacer_new_kind(const acb_table *tb, int kind, const uint8_t *rep, int64_t rep_bytes, const int64_t *rep_offsets,
                           int64_t n_ids, acb_replacer **out);

/* DEVICE buffers, asynchronous on `stream`.  The batch is laid out as for acb_scan_device; d_chosen holds the
 * *d_n_chosen <= chosen_cap records acb_leftmost_longest_device wrote for it (haystack order, then end_index ascending,
 * non-overlapping; not checked).  d_out_offsets (n_hay+1 int64 byte offsets of the output haystacks) and *d_total
 * (their total) are always written; d_out only when the total is at most out_cap, which the device checks.  d_hay and
 * d_out must be 16-byte aligned (ACB_EINVAL): the write pass reads and stores whole aligned 16-byte blocks, and may
 * read the rest of an aligned block that holds a haystack byte.  The scratch space belongs to the table: the next
 * call waits (cudaStreamWaitEvent) for the work of this one, also on another CUDA stream. */
int acb_replace_device(acb_replacer *r, acb_table *tb, const uint8_t *d_hay, int64_t total_bytes, const int64_t *d_offsets,
                       int64_t n_hay, int64_t stride_bytes, const acb_match *d_chosen, int64_t chosen_cap,
                       const int64_t *d_n_chosen, int64_t *d_out_offsets, uint8_t *d_out, int64_t out_cap, int64_t *d_total,
                       void *stream);

/* HOST buffers: upload, scan (algo ACB_ALGO_AUTO, _FILTER or _DFA) into a full list grown to fit, select, rewrite, copy
 * back, synchronous.  out_offsets and *total are always written; out when *total <= out_cap, else ACB_EOVERFLOW. */
int acb_replace_host(acb_replacer *r, acb_table *tb, const uint8_t *hay, int64_t total_bytes, const int64_t *offsets,
                     int64_t n_hay, int64_t stride_bytes, int algo, int64_t *out_offsets, uint8_t *out, int64_t out_cap,
                     int64_t *total);

/* With kernel timing on (acb_set_kernel_timing), the milliseconds of the last replacement's offsets pass and write pass
 * on this thread (the first n of them, n <= 2), from CUDA events (the call then waits for them); 0 when timing is off. */
int acb_last_replace_ms(float *ms, int32_t n);

/* ---- leftmost-longest stream batches: selection and replacement chunk by chunk ------------------------------------
 * A stream's text is the concatenation of its chunks since its start, its last reset or its last final feed.  What the
 * feeds of a stream return, concatenated, is exactly what acb_leftmost_longest_device / acb_replace_device return for
 * that whole text.  Per stream the batch keeps X, the position up to which every match is decided and emitted, and the
 * pos - X <= T = longest_word - 1 letters after it; a feed reports the chosen matches that start before
 * pos_new - T (and releases the output up to the same point), because those are the ones no later letter can change.
 * A final feed (final != 0) decides everything and returns the stream to its start: position 0, nothing held.
 * acb_streams_reset and acb_streams_positions serve these batches; acb_streams_feed_* refuse them (ACB_EINVAL), and
 * these feeds refuse the other batches.  Chunks, ids and the overflow contract are those of acb_streams_feed_*: a feed
 * that does not fit commits nothing and can be repeated.  The device feeds are asynchronous on `stream` except that
 * they wait for the staged size, the full match list's size (the full list lives in a buffer of the batch, grown to
 * fit) and, replacing, the decided windows' size.  Feeds of one batch must not overlap in time.  algo: ACB_ALGO_AUTO,
 * _FILTER or _DFA. */
int acb_streams_new_leftmost(const acb_table *tb, int64_t n_streams, acb_streams **out);

/* A leftmost stream batch of selection kind `kind`: n_bits < 0 and bits == NULL, as acb_streams_new_leftmost; else a
 * whole-word leftmost batch with that word set, as acb_streams_new_words with leftmost != 0.  Those two make batches of
 * kind ACB_SELECT_LONGEST.  The feeds select by the batch's kind; a replacing feed refuses (ACB_EINVAL) a replacer of
 * another kind. */
int acb_streams_new_leftmost_kind(const acb_table *tb, int64_t n_streams, int kind, const uint32_t *bits, int64_t n_bits,
                                  acb_streams **out);

/* The chosen records in chunk order, then end_index ascending; end_index is relative to the chunk (>= -T: a match may
 * start in letters held back from earlier chunks).  Zeroes *d_count itself, counts every chosen record, stores the
 * first cap. */
int acb_streams_feed_leftmost_device(acb_streams *ss, acb_table *tb, const uint8_t *d_chunks, int64_t total_bytes,
                                     const int64_t *d_offsets, int64_t n_chunks, int64_t stride_bytes, const int32_t *d_ids,
                                     int final, acb_match *d_out, int64_t cap, int64_t *d_count, void *stream, int algo);

/* HOST buffers: ids and offsets checked (ACB_EINVAL) before anything runs; ACB_EOVERFLOW with the exact count when the
 * records do not fit cap.  out == NULL works as for acb_scan_host (acb_copy_records / acb_take_records). */
int acb_streams_feed_leftmost_host(acb_streams *ss, acb_table *tb, const uint8_t *chunks, int64_t total_bytes,
                                   const int64_t *offsets, int64_t n_chunks, int64_t stride_bytes, const int32_t *ids, int final,
                                   acb_match *out, int64_t cap, int64_t *n_found, int algo);

/* The replacing feed: per chunk, the stream's decided text [X, X_new) with every chosen match replaced as by
 * acb_replace_device.  d_out_offsets (n_chunks+1 int64) and *d_total are always written; d_out only when the total is at
 * most out_cap (checked on the device), and only then does the feed commit.  d_out must be 16-byte aligned. */
int acb_streams_replace_device(acb_streams *ss, acb_replacer *r, acb_table *tb, const uint8_t *d_chunks, int64_t total_bytes,
                               const int64_t *d_offsets, int64_t n_chunks, int64_t stride_bytes, const int32_t *d_ids, int final,
                               int64_t *d_out_offsets, uint8_t *d_out, int64_t out_cap, int64_t *d_total, void *stream, int algo);

/* HOST buffers: out_offsets and *total are always written; out when *total <= out_cap, else ACB_EOVERFLOW. */
int acb_streams_replace_host(acb_streams *ss, acb_replacer *r, acb_table *tb, const uint8_t *chunks, int64_t total_bytes,
                             const int64_t *offsets, int64_t n_chunks, int64_t stride_bytes, const int32_t *ids, int final, int algo,
                             int64_t *out_offsets, uint8_t *out, int64_t out_cap, int64_t *total);

/* With kernel timing on, the milliseconds of the last leftmost feed's stages on this thread: staging gather, scan,
 * frontier filter, selection, window gather (replacing feeds), commit (the first n, n <= 6); 0 when timing is off.
 * acb_last_replace_ms gives a replacing feed's offsets and write passes. */
int acb_last_stream_leftmost_ms(float *ms, int32_t n);

/* ---- whole words: keep the matches that are not part of a longer word ---------------------------------------------
 * A match with end e and start s = e - len + 1 (letters) is a whole-word match iff s == 0 or letter s-1 is not a word
 * letter, and e is the haystack's last letter or letter e+1 is not a word letter.  A haystack edge counts as a non-word
 * letter: a neighbour is never read from another haystack.  The key's own letters do not matter.  A word set is a bitmap
 * of uint32 words over letter values, as the buffer stores them: letter v is a word letter iff v < n_bits and bit v
 * (bits[v / 32] >> (v % 32) & 1) is set.  n_bits is at most 256, 65 536 or 0x110000 for 1-, 2- or 4-byte letters
 * (ACB_EINVAL beyond); bits == NULL with n_bits == 0 is the set without word letters, which keeps every match. */

/* DEVICE buffers, asynchronous on `stream`.  The batch is laid out as for acb_scan_device, but d_hay needs no alignment;
 * d_records holds n records of it (what acb_scan_device leaves; hay_id, end_index and key_id are not checked), d_bits
 * the word set.  The whole-word records go to d_out in their order in d_records, from index *d_count on; *d_count is
 * increased by their number and only records below index cap are stored, as for acb_leftmost_longest_device.  d_records
 * is not changed.  The scratch space belongs to the table: the next call waits (cudaStreamWaitEvent) for the work of this
 * one, also on another CUDA stream.  ACB_ERANGE for more than 2^31-1 records. */
int acb_word_filter_device(acb_table *tb, const uint8_t *d_hay, int64_t total_bytes, const int64_t *d_offsets, int64_t n_hay,
                           int64_t stride_bytes, const acb_match *d_records, int64_t n, const uint32_t *d_bits, int64_t n_bits,
                           acb_match *d_out, int64_t cap, int64_t *d_count, void *stream);

/* HOST buffers, the word set a host bitmap: acb_scan_host, acb_scan_host_leftmost and acb_replace_host on the whole-word
 * matches only.  Each uploads the batch and scans it into a full list (algo ACB_ALGO_AUTO, _FILTER or _DFA; monolithic,
 * no pipeline), filters that list on the device, then goes on as its route does: sort (sort != 0) and copy back; select;
 * select and rewrite.  The result contracts are those routes' (ACB_EOVERFLOW with the exact count; out == NULL as for
 * acb_scan_host).  The offsets are checked (ACB_EINVAL) before anything runs.  Without a device: ACB_ECUDA. */
int acb_scan_host_words(acb_table *tb, const uint8_t *hay, int64_t total_bytes, const int64_t *offsets, int64_t n_hay,
                        int64_t stride_bytes, const uint32_t *bits, int64_t n_bits, acb_match *out, int64_t cap, int64_t *n_found,
                        int algo, int sort);
int acb_scan_host_leftmost_words(acb_table *tb, const uint8_t *hay, int64_t total_bytes, const int64_t *offsets, int64_t n_hay,
                                 int64_t stride_bytes, const uint32_t *bits, int64_t n_bits, acb_match *out, int64_t cap,
                                 int64_t *n_found, int algo);
int acb_replace_host_words(acb_replacer *r, acb_table *tb, const uint8_t *hay, int64_t total_bytes, const int64_t *offsets,
                           int64_t n_hay, int64_t stride_bytes, const uint32_t *bits, int64_t n_bits, int algo, int64_t *out_offsets,
                           uint8_t *out, int64_t out_cap, int64_t *total);

/* With kernel timing on (acb_set_kernel_timing), the milliseconds of the last whole-word filter on this thread, from its
 * flags to its count, from CUDA events (the call then waits for them); 0 when timing is off or it had no records. */
int acb_last_words_ms(float *ms);

/* ---- whole-word stream batches: find_all, leftmost-longest and replacing streams, chunk by chunk ------------------
 * A stream's text is the concatenation of its chunks since its start, its last reset or its last final feed.  Per
 * stream the batch keeps the position, up to T + 1 held letters (T = longest_word - 1) and one byte: whether the letter
 * just before the held ones exists and is a word letter.  The word set (host bitmap, as for acb_scan_host_words; checked
 * against the letter width, ACB_EINVAL) is uploaded once and belongs to the batch.
 *  - leftmost != 0: acb_streams_feed_leftmost_* and acb_streams_replace_* take the batch.  Over all feeds of a stream
 *    they return what acb_scan_host_leftmost_words / acb_replace_host_words return for its whole text; a feed reports
 *    the chosen whole-word matches that start before pos_new - T - 1 and releases the output up to there.
 *  - leftmost == 0: acb_streams_feed_words_* take the batch.  Over all feeds of a stream they return what
 *    acb_scan_host_words (sorted) returns for its whole text; a feed reports the whole-word matches that end in
 *    [pos_old - 1, pos_new - 2] (pos_new - 1 on a final feed), because a match is a whole word only once the letter after
 *    it is known.
 * A final feed decides everything and returns the stream to its start.  acb_streams_reset and acb_streams_positions
 * serve these batches; acb_streams_feed_* refuse them (ACB_EINVAL), and each feed refuses the batches of the other kind.
 * The overflow contract, the waits and the rules on streams are those of the leftmost feeds.  Without a device:
 * ACB_ECUDA. */
int acb_streams_new_words(const acb_table *tb, int64_t n_streams, int leftmost, const uint32_t *bits, int64_t n_bits,
                          acb_streams **out);

/* The whole-word records in chunk order, then end_index ascending, then longest key first; end_index is relative to the
 * chunk (>= -1: the letter after a match may arrive a feed later).  Arguments and count as acb_streams_feed_leftmost_*;
 * the host entry checks ids and offsets (ACB_EINVAL) before anything runs, and returns ACB_EOVERFLOW with the exact
 * count when the records do not fit cap. */
int acb_streams_feed_words_device(acb_streams *ss, acb_table *tb, const uint8_t *d_chunks, int64_t total_bytes,
                                  const int64_t *d_offsets, int64_t n_chunks, int64_t stride_bytes, const int32_t *d_ids,
                                  int final, acb_match *d_out, int64_t cap, int64_t *d_count, void *stream, int algo);
int acb_streams_feed_words_host(acb_streams *ss, acb_table *tb, const uint8_t *chunks, int64_t total_bytes,
                                const int64_t *offsets, int64_t n_chunks, int64_t stride_bytes, const int32_t *ids, int final,
                                acb_match *out, int64_t cap, int64_t *n_found, int algo);

/* ---- ASCII case-insensitive matching: scans of folded text -------------------------------------------------------
 * A folded table matches keys and text with every ASCII capital made small: a letter whose VALUE is 0x41..0x5A (the
 * whole letter value: a 4-byte letter U+0141 or U+1F641 is not one) reads as value + 0x20.  Nothing else folds (bytes
 * 0x80..0xFF and non-ASCII code points stay as they are), so positions and lengths are those of the text.  The trie
 * holds the folded keys, each under its group's representative: the lowest id among the keys that fold to the same
 * text.  The alias lists name the group's other ids: alias_ids[alias_ptr[k] .. alias_ptr[k+1]) for representative k,
 * ascending and above k; alias_ptr has n_keys + 1 entries (n_keys of the trie's flat view), from 0 to n_alias.  Both
 * may be NULL with n_alias == 0, the key set without case variants.  ACB_EINVAL for lists that break these rules or for
 * a trie of 2-byte letters.  An alias id has its representative's length; the table's key ids cover the aliases.
 *
 * On a folded table, acb_scan_device and every host route that scans (acb_scan_host, acb_scan_host_words, the leftmost
 * and replacement routes, plain and whole-word) fold the text before the scan: acb_scan_device into a scratch copy it
 * owns (guarded as the other scratch buffers are: the next call waits for this one's work), the pipelined acb_scan_host
 * each 32 MiB chunk in place on the device.  The word tests and the rewrites read the caller's text as it is.  Records
 * carry representative ids.  acb_scan_host and acb_scan_host_words on a table with aliases expand them before the sort
 * (acb_expand_aliases_device; such a table is not pipelined); the leftmost and replacement routes do not: the
 * representative is the leftmost-first winner and the leftmost-longest one among keys of one text.  Refused (ACB_EINVAL):
 * ACB_ALGO_LONG, the white-space scans (*_skip), the stream batch constructors other than acb_streams_new_folded (and
 * every feed of a batch they made), lookups and key selections (acb_lookup_*, acb_select_*, acb_table_upload_key_ranges).
 * A table from acb_table_upload behaves as before. */
int acb_table_upload_folded(const acb_trie *t, int device, const int32_t *alias_ptr, const int32_t *alias_ids, int64_t n_alias,
                            acb_table **out);

/* ---- case-insensitive matching through a letter map (the package's Unicode simple case folding) -------------------
 * acb_table_upload_folded with the fold given as a map: letter map_from[j] reads as map_to[j], every other letter as
 * itself.  The trie, the alias lists and everything the folded table does (scans, expansion, refusals, streams through
 * acb_streams_new_folded) are as for acb_table_upload_folded; only the fold differs.  The map's rules (ACB_EINVAL
 * otherwise): map_from strictly ascending and below 0x110000, map_to[j] < map_from[j], no map_to value among map_from
 * (the fold is idempotent), and on a trie of 1-byte letters every map_from below 256 maps below 256 (entries from 256 up
 * do not apply to 1-byte letters).  4-byte letters from 0x110000 up (not code points) read as themselves.  A 4-byte map
 * may change letters in at most 42 blocks of 256 code points (Unicode 15's simple folding uses 24); a 2-byte trie is
 * refused.  The fold is one kernel per scan with the map staged in shared memory (DESIGN section 4.19).  A stream batch
 * made on one fold refuses a table of the other (ACB_EINVAL).  Both may be NULL with n_map == 0: nothing folds. */
int acb_table_upload_folded_map(const acb_trie *t, int device, const int32_t *alias_ptr, const int32_t *alias_ids,
                                int64_t n_alias, const uint32_t *map_from, const uint32_t *map_to, int64_t n_map,
                                acb_table **out);

/* DEVICE buffers, asynchronous on `stream`; a folded table only (ACB_EINVAL).  Each of the n records of d_in becomes its
 * own record followed by one per alias of its key id, ascending (key ids without aliases, or outside the lists, stay
 * one record), at d_out in d_in's order; *d_count is SET to their total and only records below index cap are stored.
 * d_in and d_out must not overlap.  A sort of the result by acb_sort_matches_device keeps the members of a group in
 * ascending id (the radix sort is stable).  The scratch space belongs to the table, as for acb_word_filter_device.
 * ACB_ERANGE for n >= 2^31-1 (its exclusive sum runs over n + 1 counts), before anything is allocated or launched. */
int acb_expand_aliases_device(acb_table *tb, const acb_match *d_in, int64_t n, acb_match *d_out, int64_t cap, int64_t *d_count,
                              void *stream);

/* A case-folded stream batch: every stream's text matched as a folded table's scans match a whole haystack.  tb must
 * come from acb_table_upload_folded (else ACB_EINVAL).  leftmost = 0: a find_all batch, fed by acb_streams_feed_device /
 * _host, or with a word set by acb_streams_feed_words_*; leftmost = 1: a leftmost batch of selection `kind`
 * (ACB_SELECT_LONGEST or ACB_SELECT_FIRST; checked in both cases), fed by acb_streams_feed_leftmost_* and
 * acb_streams_replace_*, with or without a word set.  bits / n_bits: the word set, as for acb_streams_new_words; no word
 * set is bits == NULL with n_bits < 0.  No long mode and no skip set.  Each feed reports and releases exactly what the
 * same feed of a batch from acb_streams_new / _new_words / _new_leftmost_kind reports over the folded text (the fold maps
 * each letter alone, so folding chunk by chunk folds the stream), with the word tests and the rewrites on the text as
 * given: held letters keep their case.  A find_all feed reports every alias of each key found, after it and ascending, and
 * the capacity test of the feed is on that expanded count: a feed that overflows still changes no stream.  On a key set
 * with aliases the plain find_all feed waits once for the unexpanded count; without aliases it stays asynchronous.  The
 * feeds of a folded batch refuse any other table, and the feeds of any other batch refuse a folded table (ACB_EINVAL).
 * The device find_all feed folds into a copy the batch owns; the host feeds fold their upload in place: caller memory is
 * never written.  A find_all feed refuses what acb_scan_device refuses (ACB_ERANGE for a fixed stride past 2^31-1
 * letters) before it folds or launches anything, as the plain feed does. */
int acb_streams_new_folded(const acb_table *tb, int64_t n_streams, int leftmost, int kind, const uint32_t *bits, int64_t n_bits,
                           acb_streams **out);

/* With kernel timing on (acb_set_kernel_timing), the milliseconds of the last fold of acb_scan_device or of a folded
 * find_all stream feed (the pipelined acb_scan_host's folds are not timed) and of the last alias expansion on this thread
 * (the first n of them, n <= 2), from CUDA events (the call then waits for them); 0 when timing is off, and a folded stream
 * feed zeroes both before it runs. */
int acb_last_fold_ms(float *ms, int32_t n);

/* ---- UTF-8 batches: decoded to letters on the GPU, letters encoded back (DESIGN section 4.20) ----------------------
 * A batch of UTF-8 haystacks (d_in, 16-byte aligned: d_offsets' n_hay + 1 int64 byte offsets, any values, or rows of
 * stride_bytes with d_offsets NULL) becomes letters of 1 or 4 bytes in two passes.  A byte starts a letter unless it is
 * a continuation byte (0x80-0xBF) that the nearest other byte at most 3 bytes before it, in its haystack, covers with its
 * maximal valid prefix (Unicode Table 3-7: the second byte narrowed after E0, ED, F0 and F4; C0, C1 and F5-FF never
 * lead; never past the haystack's end).  A letter whose maximal prefix is not a whole sequence is invalid and decodes to
 * U+FFFD.  Per haystack that is CPython's bytes.decode("utf-8", "replace"); the first invalid letter is the strict
 * error, from the letter's first byte to the end of its prefix.  DEVICE buffers, asynchronous on `stream`, on `device`.
 *
 * acb_utf8_work_bytes: the workspace a batch of total_bytes and n_hay haystacks needs, for the decode and for an encode
 * of n_hay haystacks.  acb_utf8_decode_device (pass 1, two launches) fills the workspace and d_info[5]: letters in the
 * batch, largest letter, longest haystack in letters, and the first invalid letter's byte start and end in the batch
 * (-1 and -1 when there is none or errors is ACB_UTF8_REPLACE).  acb_utf8_write_device (pass 2, one launch; the same
 * batch and workspace, after the decode) stores every letter at `width` (1 or 4) bytes from d_out (16-byte aligned, room
 * for width * letters bytes; width 1 needs every letter below 256) and d_out_offsets[n_hay + 1] in output bytes.
 * acb_utf8_encode_device: letters of `width` bytes in d_in at d_offsets' byte offsets (n_hay + 1, multiples of width,
 * as acb_replace_device writes them) -> UTF-8: *d_total and d_out_offsets[n_hay + 1] always written, d_out when
 * *d_total <= out_cap (checked on the device); surrogates encode to 3 bytes and letters from 0x110000 up to U+FFFD.
 * Two launches, one with out_cap 0.  ACB_EINVAL for NULL buffers with non-zero sizes, a width other than 1 or 4, an
 * errors kind other than these two, a workspace smaller than acb_utf8_work_bytes gives, or an unaligned buffer;
 * ACB_ERANGE for more than 2^31 - 2 haystacks. */
enum { ACB_UTF8_STRICT = 0, ACB_UTF8_REPLACE = 1 };
int acb_utf8_work_bytes(int64_t total_bytes, int64_t n_hay, int64_t *bytes);
int acb_utf8_decode_device(int device, const uint8_t *d_in, int64_t total_bytes, const int64_t *d_offsets, int64_t n_hay,
                           int64_t stride_bytes, int errors, void *d_work, int64_t work_bytes, int64_t *d_info, void *stream);
int acb_utf8_write_device(int device, const uint8_t *d_in, int64_t total_bytes, const int64_t *d_offsets, int64_t n_hay,
                          int64_t stride_bytes, const void *d_work, int64_t work_bytes, int width, uint8_t *d_out,
                          int64_t *d_out_offsets, void *stream);
int acb_utf8_encode_device(int device, const uint8_t *d_in, int64_t total_bytes, const int64_t *d_offsets, int64_t n_hay,
                           int width, void *d_work, int64_t work_bytes, uint8_t *d_out, int64_t out_cap,
                           int64_t *d_out_offsets, int64_t *d_total, void *stream);

/* With kernel timing on (acb_set_kernel_timing), the milliseconds of the last UTF-8 decode pass 1, pass 2 and encode on
 * this thread (the first n, n <= 3), from CUDA events made for the call (which then waits for them); 0 when timing is off. */
int acb_last_utf8_ms(float *ms, int32_t n);

/* ---- UTF-8 stream carries: the unfinished letter of each UTF-8 stream, kept on the GPU (DESIGN section 4.21) -------
 * An acb_utf8_carry holds, per stream of a stream batch, the bytes (0 to 3) that begin a letter the stream's text has
 * not finished yet: one 32-bit word in HBM, bytes 0..2 the held bytes and byte 3 their number.  It is separate from the
 * acb_streams it serves; the caller feeds both with the same ids.  A UTF-8 feed is:
 *  1. acb_utf8_carry_stage_device: per chunk h of stream s = ids[h] (ids NULL: s = h), stage carry_s || chunk_h without
 *     its new held tail k_h into a ragged batch (d_staged at d_staged_offsets[n_chunks + 1] byte offsets), and stage
 *     the new carry, the last k_h bytes of carry_s || chunk_h.  k_h is the length from the last non-continuation byte
 *     among the last 3 bytes to the end, when that byte's maximal valid prefix (the rule of acb_utf8_decode_device)
 *     runs to the end and is shorter than its sequence, or when the text ends in ED A0-BF; else 0.  So a valid but
 *     unfinished letter is held back and a prefix that cannot be continued (E0 80, F0 8F, F4 90, C0, F5) is not: this
 *     is the buffer CPython's incremental UTF-8 decoder keeps, which also waits for the third byte after ED A0-BF.  final != 0 (the stream's text ends here): k_h = 0, so the decode reads a held prefix as
 *     the end of a haystack, as the decoder's final=True does.  Bytes from d_staged_offsets[n_chunks] up to total_bytes +
 *     3 * n_chunks (the "span", at most what the staged batch can need) are set to zero, so the decode can take the span
 *     as total_bytes without waiting for the staged size: the zeros come after the last haystack and belong to none.
 *  2. acb_utf8_decode_device / acb_utf8_write_device on (d_staged, span, d_staged_offsets, n_chunks, 0).
 *  3. a stream feed of the decoded letters, with their offsets.
 *  4. acb_utf8_carry_commit_device, once that feed has succeeded: the staged carries become the streams' carries.
 * A stage without a commit changes no carry, and a second stage restages from the committed carries.  The commit takes
 * the ids and chunk count of the last stage (ACB_EINVAL otherwise).  Streams without a chunk keep their carry.
 * Chunks as for acb_utf8_decode_device (d_chunks 16-byte aligned; d_offsets, any non-decreasing values, or rows of
 * stride_bytes); d_ids int32 device ids, distinct and in range (not checked).  d_staged 16-byte aligned with staged_cap
 * >= total_bytes + 3 * n_chunks.  Stage and commit are asynchronous on `stream`, on the carry's device.
 * ACB_EINVAL for NULL buffers with non-zero sizes, n_chunks > n_streams, a fixed stride that does not fit, a staged
 * buffer too small, an unaligned buffer; ACB_ERANGE for more than 2^31 - 2 chunks. */
typedef struct acb_utf8_carry acb_utf8_carry;
int  acb_utf8_carry_new(int device, int64_t n_streams, acb_utf8_carry **out);
void acb_utf8_carry_free(acb_utf8_carry *c);
/* ids[0..n) (host ids, in range: ACB_EINVAL otherwise; ids NULL: every stream) hold nothing.  Synchronises. */
int  acb_utf8_carry_reset(acb_utf8_carry *c, const int32_t *ids, int64_t n);
/* out[s] = the bytes stream s holds (0 to 3), cap >= n_streams.  Synchronises. */
int  acb_utf8_carry_pending(acb_utf8_carry *c, int64_t *out, int64_t cap);
/* the bytes stream `id` holds: *n of them in out[0..3).  Synchronises. */
int  acb_utf8_carry_bytes(acb_utf8_carry *c, int32_t id, uint8_t *out, int32_t *n);
int  acb_utf8_carry_stage_device(acb_utf8_carry *c, const uint8_t *d_chunks, int64_t total_bytes, const int64_t *d_offsets,
                                 int64_t n_chunks, int64_t stride_bytes, const int32_t *d_ids, int final, uint8_t *d_staged,
                                 int64_t staged_cap, int64_t *d_staged_offsets, void *stream);
int  acb_utf8_carry_commit_device(acb_utf8_carry *c, const int32_t *d_ids, int64_t n_chunks, void *stream);

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
