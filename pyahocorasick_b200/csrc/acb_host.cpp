/*
 * acb_host.cpp -- host side of the H100 Aho-Corasick path: trie arena, failure
 * links, flattening to int32 tables, gram-filter construction.
 *
 * Not a port of the reference's node graph (src/trienode.h:19-42: one malloc per
 * node, unsorted (letter, child*) pairs scanned linearly).  Here nodes live in one
 * arena with int32 ids, edges in one open-addressing hash map keyed (node, byte),
 * and the automaton is emitted as column-major int32 tables ready for upload.
 *
 * Behaviour that must equal the reference's is cited inline (paths relative to
 * /root/reference).
 */
#include "acb_internal.h"
#include "acb_hash.h"

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <exception>
#include <new>
#include <vector>
#include <wctype.h>

/* ------------------------------------------------------------------ errors */
static thread_local char g_err[512] = "";

extern "C" void acb_set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
extern "C" const char *acb_last_error(void) { return g_err; }
extern "C" int acb_abi_version(void) { return ACB_ABI_VERSION; }

/* ---------------------------------------------------------------- edge map */
namespace {

struct EdgeMap {                     /* (node << 8 | byte) -> child, open addressing */
    std::vector<uint64_t> keys;      /* 0 = empty; stored key = real key + 1 */
    std::vector<int32_t>  vals;
    size_t mask = 0, used = 0;

    static inline uint64_t mix(uint64_t x) {
        x ^= x >> 33; x *= 0xff51afd7ed558ccdULL; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ULL; x ^= x >> 33;
        return x;
    }
    void init(size_t cap_pow2) {
        keys.assign(cap_pow2, 0);
        vals.assign(cap_pow2, -1);
        mask = cap_pow2 - 1;
        used = 0;
    }
    void grow() {
        std::vector<uint64_t> ok;
        std::vector<int32_t> ov;
        ok.swap(keys);
        ov.swap(vals);
        init(ok.size() * 2);
        for (size_t i = 0; i < ok.size(); i++)
            if (ok[i]) put_raw(ok[i], ov[i]);
    }
    void put_raw(uint64_t k1, int32_t v) {
        size_t i = mix(k1) & mask;
        while (keys[i]) i = (i + 1) & mask;
        keys[i] = k1;
        vals[i] = v;
        used++;
    }
    int32_t get(int32_t node, uint8_t byte) const {
        if (keys.empty()) return -1;
        uint64_t k1 = (((uint64_t)(uint32_t)node << 8) | byte) + 1;
        size_t i = mix(k1) & mask;
        while (keys[i]) {
            if (keys[i] == k1) return vals[i];
            i = (i + 1) & mask;
        }
        return -1;
    }
    void put(int32_t node, uint8_t byte, int32_t child) {
        if (keys.empty()) init(1024);
        if ((used + 1) * 10 > keys.size() * 6) grow();
        put_raw((((uint64_t)(uint32_t)node << 8) | byte) + 1, child);
    }
};

struct Node {
    int32_t parent;
    int32_t first_child;
    int32_t last_child;
    int32_t next_sibling;
    int32_t key_id;        /* -1 = not the end of a key ("eow" false) */
    int32_t live_below;    /* live keys ending at or below this node; 0 = pruned */
    uint32_t birth;        /* stamp of the moment the link to this node was (last) made: the reference appends a child to
                              its parent's array then (src/trienode.c:125-147) and deletes it again when no key is left below
                              (src/trie.c:66-136), so this orders siblings the way its traversals see them */
    uint8_t byte;
    uint8_t n_children;    /* saturates at 255; children beyond the kListed-th are also in the edge table */
};

struct Flat {
    bool valid = false;
    int32_t S = 0, K = 0, n_keys = 0;
    int32_t min_key_bytes = 0, max_key_bytes = 0;
    uint8_t byte_class[256];
    std::vector<int32_t> goto_cm, fail, letter_fail, key_of, out_ptr, out_idx, key_len;
    int32_t gram = 0, stride = 0, log1 = 0, log3 = 0, logA = 0, filter_flags = 0, log2b = 0;
    std::vector<uint32_t> bm1, bm3, anchors;
};

} // namespace

struct acb_trie {
    int letter_bytes = 1;
    int kind = ACB_EMPTY;
    int64_t count = 0;          /* live keys */
    int64_t longest = 0;        /* letters; like the reference it never shrinks on removal */
    int64_t live_nodes = 0;     /* nodes with live_below > 0, root included once it exists */
    uint32_t birth_ctr = 0;     /* Node::birth stamps */
    std::vector<Node> nodes;
    EdgeMap edges;
    Flat flat;
};

/* ------------------------------------------------------------- trie basics */
static int32_t new_node(acb_trie *t, int32_t parent, uint8_t byte) {
    Node n;
    n.parent = parent;
    n.first_child = n.last_child = n.next_sibling = -1;
    n.key_id = -1;
    n.live_below = 0;
    n.birth = ++t->birth_ctr;
    n.byte = byte;
    n.n_children = 0;
    t->nodes.push_back(n);
    return (int32_t)(t->nodes.size() - 1);
}

extern "C" acb_trie *acb_trie_new(int letter_bytes) {
    if (letter_bytes != 1 && letter_bytes != 2 && letter_bytes != 4) {
        acb_set_error("letter_bytes must be 1, 2 or 4 (got %d)", letter_bytes);
        return nullptr;
    }
    acb_trie *t = new (std::nothrow) acb_trie();
    if (!t) { acb_set_error("out of memory"); return nullptr; }
    t->letter_bytes = letter_bytes;
    return t;
}

extern "C" void acb_trie_free(acb_trie *t) { delete t; }

extern "C" int acb_trie_clear(acb_trie *t) {
    if (!t) return ACB_EINVAL;
    int lb = t->letter_bytes;
    *t = acb_trie();
    t->letter_bytes = lb;
    return ACB_OK;
}

/* child of nd along `byte`, or -1.  Most nodes have one or two children (every byte of a wide letter but the
 * first, every node of a key's private tail), and those sit next to their parent in the arena: a short walk of
 * the sibling list answers without touching the big edge table, which is only consulted for wide fan-outs. */
constexpr int kListed = 4;             /* children found by walking the sibling list; later ones through the edge table */
static inline int32_t child_of(const acb_trie *t, int32_t nd, uint8_t byte) {
    const Node &p = t->nodes[nd];
    int32_t c = p.first_child;
    const int n = p.n_children < kListed ? p.n_children : kListed;
    for (int k = 0; k < n; k++) {
        if (t->nodes[c].byte == byte) return c;
        c = t->nodes[c].next_sibling;
    }
    return p.n_children > kListed ? t->edges.get(nd, byte) : -1;
}

extern "C" int acb_trie_add_word(acb_trie *t, const uint8_t *key, int64_t nbytes, int32_t key_id,
                                 int32_t *prev_key_id) {
    if (!t || key_id < 0 || nbytes < 0 || (nbytes && !key)) { acb_set_error("bad argument"); return ACB_EINVAL; }
    if (nbytes % t->letter_bytes) { acb_set_error("key length %lld is not a multiple of letter_bytes", (long long)nbytes); return ACB_EINVAL; }
    if (nbytes == 0) {                      /* src/Automaton.c:257,295: empty key is ignored */
        if (prev_key_id) *prev_key_id = -2;
        return ACB_OK;
    }
    if (nbytes > 0x3fffffff) { acb_set_error("key too long"); return ACB_ERANGE; }
    try {
        if (t->nodes.empty()) { new_node(t, -1, 0); t->live_nodes = 1; }   /* root, src/trie.c:21-26 */
        int32_t nd = 0;
        for (int64_t i = 0; i < nbytes; i++) {
            int32_t kid = child_of(t, nd, key[i]);
            if (kid < 0) {
                if (t->nodes.size() >= 0x7ffffff0u) { acb_set_error("too many trie nodes for int32 state ids"); return ACB_ERANGE; }
                kid = new_node(t, nd, key[i]);
                Node &p = t->nodes[nd];
                if (p.last_child < 0) p.first_child = kid; else t->nodes[p.last_child].next_sibling = kid;
                p.last_child = kid;
                if (p.n_children >= kListed) t->edges.put(nd, key[i], kid);   /* the first kListed are found by the list walk */
                if (p.n_children < 255) p.n_children++;
            }
            nd = kid;
        }
        int32_t prev = t->nodes[nd].key_id;
        t->nodes[nd].key_id = key_id;
        if (prev < 0) {                                      /* a new key: src/trie.c:52-56 */
            t->count += 1;
            for (int32_t x = nd; x >= 0; x = t->nodes[x].parent) {
                if (x != 0 && t->nodes[x].live_below == 0) {                     /* the root is always live */
                    t->live_nodes += 1;
                    t->nodes[x].birth = ++t->birth_ctr;                          /* (re)linked now: last among its siblings */
                }
                t->nodes[x].live_below += 1;
            }
            int64_t letters = nbytes / t->letter_bytes;      /* src/Automaton.c:285-286 */
            if (letters > t->longest) t->longest = letters;
        }
        t->kind = ACB_TRIE;                                  /* src/trie.c:60 -- also demotes AHOCORASICK */
        t->flat.valid = false;
        if (prev_key_id) *prev_key_id = prev;
        return ACB_OK;
    } catch (const std::bad_alloc &) {
        acb_set_error("out of memory");
        return ACB_ENOMEM;
    } catch (const std::exception &e) {
        acb_set_error("add_word: %s", e.what());
        return ACB_ERANGE;
    }
}

static int32_t walk(const acb_trie *t, const uint8_t *key, int64_t nbytes, int64_t *consumed) {
    int32_t nd = t->nodes.empty() ? -1 : 0;
    int64_t i = 0;
    for (; nd >= 0 && i < nbytes; i++) {
        int32_t kid = child_of(t, nd, key[i]);
        if (kid < 0 || t->nodes[kid].live_below == 0) break;
        nd = kid;
    }
    if (consumed) *consumed = i;
    return (i == nbytes) ? nd : -1;
}

extern "C" int acb_trie_find(const acb_trie *t, const uint8_t *key, int64_t nbytes, int32_t *key_id,
                             int32_t *is_prefix) {
    if (!t || nbytes < 0) return ACB_EINVAL;
    int32_t nd = walk(t, key, nbytes, nullptr);
    if (key_id) *key_id = (nd >= 0 && nbytes > 0) ? t->nodes[nd].key_id : -1;
    if (is_prefix) *is_prefix = (nd >= 0) ? 1 : 0;
    return ACB_OK;
}

extern "C" int64_t acb_trie_longest_prefix(const acb_trie *t, const uint8_t *key, int64_t nbytes) {
    if (!t || nbytes < 0) return 0;
    int64_t used = 0;
    walk(t, key, nbytes, &used);
    return used / t->letter_bytes;      /* only whole letters count */
}

extern "C" int acb_trie_remove_word(acb_trie *t, const uint8_t *key, int64_t nbytes, int32_t *key_id) {
    if (!t || nbytes < 0) return ACB_EINVAL;
    if (key_id) *key_id = -1;
    if (nbytes == 0) return ACB_OK;
    int32_t nd = walk(t, key, nbytes, nullptr);
    if (nd < 0 || t->nodes[nd].key_id < 0) return ACB_OK;
    if (key_id) *key_id = t->nodes[nd].key_id;
    t->nodes[nd].key_id = -1;
    t->count -= 1;
    for (int32_t x = nd; x >= 0; x = t->nodes[x].parent) {
        t->nodes[x].live_below -= 1;
        if (x != 0 && t->nodes[x].live_below == 0) t->live_nodes -= 1;
    }
    t->kind = ACB_TRIE;                  /* src/trie.c:134 -- stays TRIE even when no key is left */
    t->flat.valid = false;
    return ACB_OK;
}

extern "C" int acb_trie_kind(const acb_trie *t) { return t ? t->kind : ACB_EMPTY; }
extern "C" int64_t acb_trie_count(const acb_trie *t) { return t ? t->count : 0; }
extern "C" int64_t acb_trie_longest_word(const acb_trie *t) { return t ? t->longest : 0; }
extern "C" int64_t acb_trie_nodes(const acb_trie *t) { return t ? t->live_nodes : 0; }
extern "C" int64_t acb_trie_links(const acb_trie *t) { return (t && t->live_nodes > 0) ? t->live_nodes - 1 : 0; }
extern "C" int64_t acb_trie_host_bytes(const acb_trie *t) {
    if (!t) return 0;
    return (int64_t)(t->nodes.capacity() * sizeof(Node) + t->edges.keys.capacity() * (sizeof(uint64_t) + sizeof(int32_t)));
}

/* ---------------------------------------------------------- gram filter */
namespace {

/* ACB_TRACE=1: phase times of make_automaton on stderr */
struct PhaseTimer {
    bool on;
    std::chrono::steady_clock::time_point t0;
    PhaseTimer() : on(getenv("ACB_TRACE") != nullptr), t0(std::chrono::steady_clock::now()) {}
    void lap(const char *what) {
        if (!on) return;
        auto t1 = std::chrono::steady_clock::now();
        fprintf(stderr, "[make_automaton] %-28s %8.1f ms\n", what, std::chrono::duration<double, std::milli>(t1 - t0).count());
        t0 = t1;
    }
};

struct FilterChoice {
    int g = 0, s = 0, log1 = 0;
    double cost = 1e300;
};

static inline void set_bit(std::vector<uint32_t> &bm, uint32_t idx) { bm[idx >> 5] |= 1u << (idx & 31); }

/* a gram (g <= 16 bytes) as two zero-padded little-endian words: cheap to copy, sort and compare */
struct Gram16 {
    uint64_t a = 0, b = 0;
    const uint8_t *data() const { return reinterpret_cast<const uint8_t *>(this); }
    bool operator<(const Gram16 &o) const { return a != o.a ? a < o.a : b < o.b; }
    bool operator==(const Gram16 &o) const { return a == o.a && b == o.b; }
};
static inline Gram16 load_gram(const uint8_t *p, int g) {
    Gram16 x;
    memcpy(&x, p, (size_t)g);
    return x;
}
static inline uint64_t mix_gram(const Gram16 &x) {
    uint64_t h = x.a * 0x9E3779B97F4A7C15ULL ^ (x.b + 0xC2B2AE3D27D4EB4FULL) * 0xFF51AFD7ED558CCDULL;
    h ^= h >> 32; h *= 0xD6E8FEB86659FD93ULL; h ^= h >> 29;
    return h;
}

/* number of distinct grams of the m-prefixes at offsets 0, L, .., s-L (the cost model's E): counted over
 * 64-bit fingerprints, so the candidate shapes can be compared without materialising their gram sets */
static size_t count_grams(const std::vector<std::vector<uint8_t>> &prefixes, int g, int s, int L, std::vector<uint64_t> &scratch) {
    scratch.clear();
    for (const auto &p : prefixes)
        for (int j = 0; j + L <= s; j += L) {
            if (j + g > (int)p.size()) break;
            scratch.push_back(mix_gram(load_gram(p.data() + j, g)));
        }
    std::sort(scratch.begin(), scratch.end());
    return (size_t)(std::unique(scratch.begin(), scratch.end()) - scratch.begin());
}

/* the distinct grams themselves (for the chosen shape only) */
static void collect_grams(const std::vector<std::vector<uint8_t>> &prefixes, int g, int s, int L, std::vector<Gram16> &out) {
    out.clear();
    for (const auto &p : prefixes)
        for (int j = 0; j + L <= s; j += L) {
            if (j + g > (int)p.size()) break;
            out.push_back(load_gram(p.data() + j, g));
        }
    std::sort(out.begin(), out.end());
    out.erase(std::unique(out.begin(), out.end()), out.end());
}

static int ceil_log2_u64(uint64_t x) {
    int l = 0;
    while (((uint64_t)1 << l) < x && l < 62) l++;
    return l;
}

} // namespace

/* Gram filter + anchor table (DESIGN.md "filter kernel").
 *
 * Every occurrence of a key K at byte position p contains exactly one probe position
 * q = p + j, q a multiple of the stride s, with j in {0, L, .., s-L}; the g bytes at q are
 * K[j..j+g).  Stage 1 is a bitmap over hash1(gram) (shared memory), stage 2 a bitmap over
 * hash2(gram) (global memory).  The anchor table maps hash2(gram) to the
 * trie nodes at depth j+g whose last g bytes are that gram:
 *   - a node with exactly one key below it (and that key <= 20 bytes) becomes a UNIQUE entry
 *     carrying the key itself: the device compares the text at q-j with the key directly;
 *   - otherwise the whole (gram, j) group collapses to one MULTI entry carrying the gram: the
 *     device walks the trie from the root at q-j.
 * Entry = 8 x uint32: tag (hash2|1, 0 = empty), key_id (-1 = MULTI), j | len<<8 | last<<16 (last = no
 * further entry with this tag in the probe sequence), 20 key/gram bytes. */
static int build_filter(acb_trie *t, Flat &f) {
    PhaseTimer pt;
    const int L = t->letter_bytes;
    const int m = f.min_key_bytes;
    /* live nodes down to depth m, with depths */
    std::vector<int32_t> depth(t->nodes.size(), -1);
    std::vector<std::vector<uint8_t>> prefixes;
    {
        std::vector<int32_t> stack;
        depth[0] = 0;
        stack.push_back(0);
        while (!stack.empty()) {
            int32_t nd = stack.back();
            stack.pop_back();
            if (depth[nd] == m) {
                std::vector<uint8_t> p(m);
                int32_t x = nd;
                for (int i = m - 1; i >= 0; i--) { p[i] = t->nodes[x].byte; x = t->nodes[x].parent; }
                prefixes.push_back(std::move(p));
                continue;
            }
            for (int32_t c = t->nodes[nd].first_child; c >= 0; c = t->nodes[c].next_sibling)
                if (t->nodes[c].live_below > 0) { depth[c] = depth[nd] + 1; stack.push_back(c); }
        }
    }
    pt.lap("filter: prefixes");
    /* ACB_FILTER=g,s,log1,mode (mode 0 single, 1 pair) forces the shape, for tests and experiments; a field left out or
       given as 0 (mode: -1) stays the cost model's choice.  A shape the kernels cannot run is refused here rather
       than built: a stride that is not L * 2^k <= 16, a level 1 outside 2^13..2^20 bits, a pair placement other than
       gram 4 / stride 1 / 1-byte letters, or a gram / stride pair that this key set does not offer. */
    int forced_g = 0, forced_s = 0, forced_l1 = 0, forced_mode = -1;
    const char *forced = getenv("ACB_FILTER");
    if (forced) {
        const int n = sscanf(forced, "%d,%d,%d,%d", &forced_g, &forced_s, &forced_l1, &forced_mode);
        if (n < 1) { acb_set_error("ACB_FILTER=\"%s\": expected g,s,log1,mode", forced); return ACB_EINVAL; }
        if (forced_g < 0 || forced_g > ACB_MAX_GRAM || forced_g % L) {
            acb_set_error("ACB_FILTER: gram %d is not a multiple of %d bytes in 1..%d", forced_g, L, ACB_MAX_GRAM);
            return ACB_EINVAL;
        }
        if (forced_s && (forced_s < L || forced_s > 16 || (forced_s & (forced_s - 1)))) {
            acb_set_error("ACB_FILTER: stride %d is not %d * 2^k <= 16", forced_s, L);
            return ACB_EINVAL;
        }
        if (forced_l1 && (forced_l1 < 13 || forced_l1 > 20)) {
            acb_set_error("ACB_FILTER: log1 %d is outside 13..20", forced_l1);
            return ACB_EINVAL;
        }
        if (forced_mode < -1 || forced_mode > 1) { acb_set_error("ACB_FILTER: mode %d is neither 0 (single) nor 1 (pair)", forced_mode); return ACB_EINVAL; }
        if (forced_mode == 1 && !(forced_g == 4 && forced_s == 1 && L == 1)) {
            acb_set_error("ACB_FILTER: the pair placement needs gram 4, stride 1 and 1-byte letters (got gram %d, stride %d, %d-byte letters)",
                          forced_g, forced_s, L);
            return ACB_EINVAL;
        }
    }

    /* Pick gram length g, probe stride s and the placement (single / pair) by a small cost model, in issue
     * cycles per text byte of one SM sub-partition (DESIGN.md section 4.1): a single-position probe is bound by the
     * bank conflicts of its shared-memory load (about 17 cycles per position and warp), a pair probe by the ALU
     * pipe (about 9); every survivor of the bitmap costs an anchor-table visit in L2 and a divergent round. */
    const double Kb = std::max(1, f.K - 1);
    FilterChoice best;
    int best_pair = 0;
    double best_pass = 0;
    std::vector<Gram16> best_grams;
    std::vector<uint64_t> scratch;
    auto pass_rate = [](double lambda) {                 /* blocked Bloom, k = 2: P(both bits of a foreign gram are set) */
        double pass = 0, pn = std::exp(-lambda);         /* Poisson(n; lambda) entries in the word */
        for (int n = 1; n <= 64; n++) {
            pn *= lambda / n;
            const double bits = 32.0 * (1.0 - std::pow(1.0 - 1.0 / 32.0, 2.0 * n));   /* distinct bits set by n entries */
            pass += pn * std::min(1.0, bits * (bits - 1.0) / (32.0 * 31.0));
        }
        return pass;
    };
    for (int s = L; s <= 16; s *= 2) {
        if (forced_s && s != forced_s) continue;
        int gmax = std::min(ACB_MAX_GRAM, m - s + L);
        if (gmax < L) break;
        gmax -= gmax % L;
        std::vector<int> gs;
        gs.push_back(gmax);
        for (int g = 12; g >= 4; g -= 4) if (g < gmax && g % L == 0) gs.push_back(g);
        for (int g : gs) {
            if (forced_g && g != forced_g) continue;
            const double E = (double)count_grams(prefixes, g, s, L, scratch);
            int log1 = std::min(20, std::max(13, ceil_log2_u64((uint64_t)(E * 64.0) + 1)));
            if (forced_l1) log1 = forced_l1;
            const double words = std::pow(2.0, log1 - 5);
            const double space = std::pow(Kb, (double)g);
            const double p_true = std::min(1.0, E / space);
            const int nw = (g + 3) / 4;
            for (int pair = 0; pair <= 1; pair++) {
                if (pair && !(L == 1 && s == 1 && g == 4)) continue;
                if (forced_mode >= 0 && pair != forced_mode) continue;
                /* pair: a foreign position must find its role's bit set in level 1 (2E entries in 2^log1 bits, a little
                   more for the unevenly used five low bits of a text byte) -- it then costs an item round -- and both of
                   its tag's bits in level 2 (blocked Bloom, k = 2, 2E bits in 2^log2b) to reach the anchor table */
                const int log2b = log1 >= 20 ? 17 : std::min(19, std::max(13, log1));
                const double pass_l1 = std::min(1.0, 1.3 * 2.0 * E / (words * 32.0));
                const double fill2 = std::min(1.0, 2.0 * E / std::pow(2.0, log2b));
                const double pass1 = pair ? p_true + (1 - p_true) * pass_l1 * fill2 * fill2
                                          : p_true + (1 - p_true) * pass_rate(E / words);
                const double probe = pair ? 6.0 + 40.0 * pass_l1 : std::max(17.0, 5.0 + 3.0 * nw);
                const double cost = (probe + pass1 * 120.0 + p_true * (s / L) * 40.0) / s;
                if (cost < best.cost) {
                    best.g = g; best.s = s; best.log1 = log1; best.cost = cost;
                    best_pair = pair;
                    best_pass = pass1 - p_true;
                }
            }
        }
    }
    if (best.g == 0) {                                   /* only a forcing can leave no candidate */
        acb_set_error("ACB_FILTER=\"%s\": gram %d / stride %d is not a candidate for keys of %d bytes and more (gram + stride <= %d)",
                      forced ? forced : "", forced_g, forced_s, m, m + L);
        return ACB_EINVAL;
    }
    collect_grams(prefixes, best.g, best.s, L, best_grams);
    pt.lap("filter: choose gram/stride");
    const int g = best.g, s = best.s;
    f.gram = g;
    f.stride = s;
    f.log1 = best.log1;
    /* The bitmap: 2^log1 bits of shared memory, 2^(log1-5) words.  A gram sets two bits of ONE word (a blocked
     * Bloom filter with k = 2: the probe costs one shared-memory load, and a random gram has to find BOTH bits set).
     *   single: word = umulhi(hash1, n_words), bits acb_stage1_bit_a AND acb_stage1_bit_b (acb_hash.h);
     *   pair  : two levels in the two halves of the bits, acb_pair_place, every gram once per role. */
    const uint32_t n_words = 1u << (best.log1 - 5);
    /* pair placement: level 2 follows level 1.  Together with the ring and the candidate rings of the pair kernel a
       2^20-bit level 1 leaves 16 KiB of shared memory; a smaller level 1 leaves room for 2^19 bits */
    f.log2b = best_pair ? (best.log1 >= 20 ? 17 : std::min(19, std::max(13, best.log1))) : 0;       /* the cost model's */
    f.bm1.assign((size_t)n_words + (f.log2b ? (size_t)1 << (f.log2b - 5) : 0), 0);
    uint32_t mul1[ACB_MAX_WINDOWS], mul2[ACB_MAX_WINDOWS];
    acb_hash_multipliers(g, 1, mul1);
    acb_hash_multipliers(g, 2, mul2);
    f.filter_flags = best_pair ? ACB_FILTER_PAIR : (acb_hash_is_wide(g) ? ACB_FILTER_WIDE : 0);
    for (const auto &gr : best_grams) {
        if (best_pair) {
            const uint8_t *b = gr.data();
            const uint32_t G = (uint32_t)b[0] | ((uint32_t)b[1] << 8) | ((uint32_t)b[2] << 16) | ((uint32_t)b[3] << 24);
            for (int role = 0; role < 2; role++) {
                uint32_t word1, bit1;
                acb_pair_place(G, role, best.log1, &word1, &bit1);
                f.bm1[word1] |= bit1;
            }
            uint32_t word2, bits2;
            acb_pair_place2(acb_hash_bytes(b, g, mul2) | 1u, f.log2b, &word2, &bits2);
            f.bm1[(size_t)n_words + word2] |= bits2;
        } else {
            const uint64_t hw = acb_hash_bytes_wide(gr.data(), g, mul1);
            const uint32_t h1 = (uint32_t)hw;
            const uint32_t bits = (1u << acb_stage1_bit_a(hw, g, best.log1)) | (1u << acb_stage1_bit_b(hw));
            f.bm1[(size_t)(((uint64_t)h1 * n_words) >> 32)] |= bits;
        }
    }

    pt.lap("filter: bitmaps");
    /* ---- anchor table ---- */
    /* candidates: every live node at depth j + g (j a probe offset) with the last g bytes of its path.  One
       LIFO walk with the path kept per depth -- no parent chasing; for a node with a single key below it the key
       is read off right here (path + the one chain down to it). */
    struct Cand { Gram16 gram; int j; int32_t node; int32_t uniq; };
    struct Uniq { int32_t key_id; uint8_t len; uint8_t bytes[20]; };      /* len 255: longer than an entry can carry */
    std::vector<Cand> cands;
    std::vector<Uniq> uniqs;
    {
        std::vector<uint8_t> path((size_t)m + 1, 0);
        std::vector<int32_t> stack;
        stack.push_back(0);
        while (!stack.empty()) {
            const int32_t nd = stack.back();
            stack.pop_back();
            const int d = depth[nd];
            if (d > 0) {
                path[d - 1] = t->nodes[nd].byte;
                const int j = d - g;
                if (j >= 0 && j <= s - L && (j % L) == 0) {
                    Cand c;
                    c.gram = load_gram(&path[d - g], g);
                    c.j = j;
                    c.node = nd;
                    c.uniq = -1;
                    if (t->nodes[nd].live_below == 1) {
                        Uniq u;
                        u.key_id = -1;
                        u.len = 255;
                        uint8_t kb[20];
                        int n = 0;
                        bool fits = d <= 20;
                        if (fits) { memcpy(kb, path.data(), (size_t)d); n = d; }
                        int32_t x = nd;
                        while (fits && t->nodes[x].key_id < 0) {
                            int32_t nxt = -1;
                            for (int32_t ch = t->nodes[x].first_child; ch >= 0; ch = t->nodes[ch].next_sibling)
                                if (t->nodes[ch].live_below > 0) { nxt = ch; break; }
                            if (nxt < 0) { fits = false; break; }            /* cannot happen for live_below == 1 */
                            if (n == 20) { fits = false; break; }
                            kb[n++] = t->nodes[nxt].byte;
                            x = nxt;
                        }
                        if (fits) { u.key_id = t->nodes[x].key_id; u.len = (uint8_t)n; memcpy(u.bytes, kb, (size_t)n); }
                        c.uniq = (int32_t)uniqs.size();
                        uniqs.push_back(u);
                    }
                    cands.push_back(c);
                }
            }
            if (d < m)
                for (int32_t ch = t->nodes[nd].first_child; ch >= 0; ch = t->nodes[ch].next_sibling)
                    if (t->nodes[ch].live_below > 0) stack.push_back(ch);
        }
    }
    std::sort(cands.begin(), cands.end(), [](const Cand &a, const Cand &b) {      /* groups (j, gram); any total order will do */
        if (a.j != b.j) return a.j < b.j;
        if (!(a.gram == b.gram)) return a.gram < b.gram;
        return a.node < b.node;
    });
    struct Entry { uint32_t w[8]; };
    std::vector<Entry> entries, group;
    entries.reserve(cands.size());
    auto pack = [](Entry &e, uint32_t tag, int32_t key_id, int j, int len, const uint8_t *bytes) {
        memset(&e, 0, sizeof(e));
        e.w[0] = tag;
        e.w[1] = (uint32_t)key_id;
        e.w[2] = (uint32_t)j | ((uint32_t)len << 8);
        for (int i = 0; i < len && i < 20; i++) e.w[3 + (i >> 2)] |= (uint32_t)bytes[i] << (8 * (i & 3));
    };
    for (size_t a = 0; a < cands.size();) {
        size_t b = a;
        while (b < cands.size() && cands[b].j == cands[a].j && cands[b].gram == cands[a].gram) b++;
        uint32_t tag = acb_hash_bytes(cands[a].gram.data(), g, mul2) | 1u;
        bool multi = false;
        group.clear();
        for (size_t i = a; i < b && !multi; i++) {
            if (cands[i].uniq < 0) { multi = true; break; }                /* more than one key below the node */
            const Uniq &u = uniqs[cands[i].uniq];
            if (u.key_id < 0 || u.len > 20) { multi = true; break; }
            Entry e;
            pack(e, tag, u.key_id, cands[a].j, (int)u.len, u.bytes);
            group.push_back(e);
        }
        if (multi) {
            Entry e;
            pack(e, tag, -1, cands[a].j, g, cands[a].gram.data());
            entries.push_back(e);
        } else {
            entries.insert(entries.end(), group.begin(), group.end());
        }
        a = b;
    }
    pt.lap("filter: anchor entries");
    /* The tag bitmap: a bitmap in global memory (L2-resident) over a re-mix of the anchor tag, 64 bits per distinct tag.
     * Only built when the shared-memory filter lets more than one per cent of foreign grams through (large or very
     * repetitive key sets): it keeps that flood away from the candidate lists and the anchor table at the price of one
     * L2 access per survivor. */
    f.log3 = 0;
    f.bm3.assign(1, 0);
    if (best_pass > 0.01 || getenv("ACB_FORCE_TAGMAP")) {
        int log3 = std::min(30, std::max(16, ceil_log2_u64((uint64_t)entries.size() * 64 + 1)));
        f.log3 = log3;
        f.bm3.assign((size_t)1 << (log3 - 5), 0);
        for (const Entry &e : entries) set_bit(f.bm3, (e.w[0] * ACB_TAGMAP_MIX) >> (32 - log3));
    }
    int logA = std::max(10, ceil_log2_u64((uint64_t)entries.size() * 4 + 1));     /* load factor <= 1/4 */
    if (logA > 28) logA = 28;
    while (((size_t)1 << logA) < entries.size() + entries.size() / 4 + 1) logA++;
    f.logA = logA;
    const size_t slots = (size_t)1 << logA, mask = slots - 1;
    f.anchors.assign(slots * 8, 0);
    /* insert tag by tag; within one tag the chain order is the insertion order, and the last entry of
     * the tag gets bit 16 of word 2 set so that a lookup can stop there */
    std::stable_sort(entries.begin(), entries.end(), [](const Entry &a, const Entry &b) { return a.w[0] < b.w[0]; });
    for (size_t a = 0; a < entries.size(); a++) {
        Entry e = entries[a];
        if (a + 1 == entries.size() || entries[a + 1].w[0] != e.w[0]) e.w[2] |= 1u << 16;
        size_t i = e.w[0] >> (32 - logA);                   /* slot from the high bits of hash2 */
        while (f.anchors[i * 8] != 0) i = (i + 1) & mask;
        memcpy(&f.anchors[i * 8], e.w, sizeof(e.w));
    }
    pt.lap("filter: anchor table");
    return ACB_OK;
}

/* ----------------------------------------------- make_automaton + flatten */
extern "C" int acb_trie_make_automaton(acb_trie *t, int32_t *built) {
    if (!t) return ACB_EINVAL;
    if (built) *built = 0;
    if (t->kind != ACB_TRIE) return ACB_OK;              /* src/Automaton.c:574-575 */
    try {
        PhaseTimer pt;
        Flat &f = t->flat;
        f = Flat();
        const int64_t S64 = t->live_nodes;
        if (S64 <= 0 || S64 > 0x7ffffff0) { acb_set_error("state count out of range"); return ACB_ERANGE; }
        const int32_t S = (int32_t)S64;

        /* byte classes: 0 = byte on no edge; 1.. in byte order */
        bool present[256] = {false};
        int np = 0;
        for (size_t i = 1; i < t->nodes.size(); i++)
            if (t->nodes[i].live_below > 0 && !present[t->nodes[i].byte]) { present[t->nodes[i].byte] = true; np++; }
        int32_t K;
        if (np == 256) {
            /* every byte value occurs on some edge: no "other" class, class = byte */
            for (int b = 0; b < 256; b++) f.byte_class[b] = (uint8_t)b;
            K = 256;
        } else {
            K = 1;
            for (int b = 0; b < 256; b++) f.byte_class[b] = present[b] ? (uint8_t)K++ : (uint8_t)0;
        }
        if ((int64_t)K * S64 > ((int64_t)1 << 33)) {
            acb_set_error("goto table would need %lld entries (K=%d classes x S=%d states)", (long long)K * S64, K, S);
            return ACB_ERANGE;
        }

        /* BFS numbering (root = 0), children in insertion order */
        std::vector<int32_t> order;            /* new id -> arena id */
        std::vector<int32_t> newid(t->nodes.size(), -1);
        order.reserve(S);
        order.push_back(0);
        newid[0] = 0;
        for (size_t h = 0; h < order.size(); h++) {
            const Node &nd = t->nodes[order[h]];
            for (int32_t c = nd.first_child; c >= 0; c = t->nodes[c].next_sibling)
                if (t->nodes[c].live_below > 0) { newid[c] = (int32_t)order.size(); order.push_back(c); }
        }
        if ((int32_t)order.size() != S) { acb_set_error("internal: live node count mismatch"); return ACB_EINVAL; }

        f.S = S;
        f.K = K;
        f.goto_cm.assign((size_t)K * S, -1);
        f.fail.assign(S, 0);
        f.key_of.assign(S, -1);
        std::vector<int32_t> depth(S, 0);
        int32_t max_id = -1;
        for (int32_t s = 1; s < S; s++) {
            const Node &nd = t->nodes[order[s]];
            int32_t ps = newid[nd.parent];
            f.goto_cm[(size_t)f.byte_class[nd.byte] * S + ps] = s;
            depth[s] = depth[ps] + 1;
        }
        int32_t minb = 0x7fffffff, maxb = 0;
        for (int32_t s = 0; s < S; s++) {
            int32_t k = t->nodes[order[s]].key_id;
            f.key_of[s] = k;
            if (k >= 0) { max_id = std::max(max_id, k); minb = std::min(minb, depth[s]); maxb = std::max(maxb, depth[s]); }
        }
        f.n_keys = max_id + 1;
        if (max_id < 0) minb = 0;                            /* every key was removed: root-only automaton */
        f.min_key_bytes = minb;
        f.max_key_bytes = maxb;
        f.key_len.assign(f.n_keys, 0);
        for (int32_t s = 0; s < S; s++) if (f.key_of[s] >= 0) f.key_len[f.key_of[s]] = depth[s] / t->letter_bytes;

        /* failure links: src/Automaton.c:582-637.  BFS order guarantees fail[] of
         * shallower states is final when a state is processed. */
        f.fail[0] = -1;                                      /* root has no fail link (SURVEY A12) */
        for (int32_t s = 1; s < S; s++) {
            const Node &nd = t->nodes[order[s]];
            int32_t ps = newid[nd.parent];
            if (ps == 0) { f.fail[s] = 0; continue; }       /* depth-1 states fail to the root, :582-596 */
            const size_t col = (size_t)f.byte_class[nd.byte] * S;
            int32_t st = f.fail[ps];
            while (st != 0 && f.goto_cm[col + st] < 0) st = f.fail[st];   /* :621-629 */
            int32_t g = f.goto_cm[col + st];
            f.fail[s] = (g >= 0) ? g : 0;                                 /* :631-633 */
        }

        /* letter-level failure link (iter_long walks the trie letter by letter): the first state on the
         * byte-level fail chain that sits on a letter boundary; equal to fail[] for 1-byte letters */
        f.letter_fail.assign(S, -1);
        for (int32_t s = 1; s < S; s++) {
            if (depth[s] % t->letter_bytes) continue;
            int32_t x = f.fail[s];
            while (x > 0 && depth[x] % t->letter_bytes) x = f.fail[x];
            f.letter_fail[s] = x < 0 ? 0 : x;
        }

        /* CSR output lists: keys on s, fail(s), fail(fail(s)).. (longest first) */
        std::vector<int32_t> osuf(S, -1), cnt(S, 0);
        int64_t total = 0;
        for (int32_t s = 1; s < S; s++) {
            int32_t fl = f.fail[s];
            osuf[s] = (fl > 0) ? ((f.key_of[fl] >= 0) ? fl : osuf[fl]) : -1;
            cnt[s] = (f.key_of[s] >= 0 ? 1 : 0) + (osuf[s] >= 0 ? cnt[osuf[s]] : 0);
            total += cnt[s];
            if (total > 0x7fffffff) { acb_set_error("output lists exceed int32 (%lld entries)", (long long)total); return ACB_ERANGE; }
        }
        f.out_ptr.assign((size_t)S + 1, 0);
        for (int32_t s = 0; s < S; s++) f.out_ptr[s + 1] = f.out_ptr[s] + cnt[s];
        f.out_idx.assign((size_t)total, -1);
        for (int32_t s = 1; s < S; s++) {
            int32_t w = f.out_ptr[s];
            for (int32_t x = (f.key_of[s] >= 0) ? s : osuf[s]; x >= 0; x = osuf[x]) f.out_idx[w++] = f.key_of[x];
        }

        pt.lap("goto / fail / outputs");
        if (f.n_keys > 0) {
            const int rc = build_filter(t, f);
            if (rc != ACB_OK) { t->flat = Flat(); return rc; }
        } else {                                               /* nothing can ever match */
            f.gram = t->letter_bytes; f.stride = t->letter_bytes; f.log1 = 13; f.logA = 10; f.log3 = 0; f.bm3.assign(1, 0);
            f.filter_flags = acb_hash_is_wide(f.gram) ? ACB_FILTER_WIDE : 0;
            f.bm1.assign((size_t)1 << (13 - 5), 0);
            f.anchors.assign(((size_t)1 << 10) * 8, 0);
        }
        f.valid = true;
        t->kind = ACB_AHOCORASICK;                           /* :639 */
        if (built) *built = 1;
        return ACB_OK;
    } catch (const std::bad_alloc &) {
        t->flat = Flat();
        acb_set_error("out of memory while flattening");
        return ACB_ENOMEM;
    } catch (const std::exception &e) {                      /* std::length_error etc.: nothing may cross the C ABI */
        t->flat = Flat();
        acb_set_error("make_automaton: %s", e.what());
        return ACB_ERANGE;
    }
}

extern "C" int acb_trie_flat_view(const acb_trie *t, acb_flat_view *out) {
    if (!t || !out) return ACB_EINVAL;
    if (t->kind != ACB_AHOCORASICK || !t->flat.valid) { acb_set_error("not an Aho-Corasick automaton yet"); return ACB_ESTATE; }
    const Flat &f = t->flat;
    memset(out, 0, sizeof(*out));
    out->n_states = f.S;
    out->n_classes = f.K;
    out->n_keys = f.n_keys;
    out->letter_bytes = t->letter_bytes;
    out->min_key_bytes = f.min_key_bytes;
    out->max_key_bytes = f.max_key_bytes;
    out->byte_class = f.byte_class;
    out->goto_cm = f.goto_cm.data();
    out->fail = f.fail.data();
    out->letter_fail = f.letter_fail.data();
    out->key_of = f.key_of.data();
    out->out_ptr = f.out_ptr.data();
    out->out_idx = f.out_idx.data();
    out->key_len = f.key_len.data();
    out->gram_bytes = f.gram;
    out->stride = f.stride;
    out->log2_bits1 = f.log1;
    out->log2_anchor_slots = f.logA;
    out->log2_bits3 = f.log3;
    out->bitmap3 = f.bm3.data();
    out->bitmap1 = f.bm1.data();
    out->anchors = f.anchors.data();
    out->filter_flags = f.filter_flags;
    out->log2_bits2 = f.log2b;
    return ACB_OK;
}

/* ------------------------------------------------ the flat-table cache (include/acb200.h) */
namespace {

constexpr char kFlatMagic[8] = {'A', 'C', 'B', 'F', 'L', 'A', 'T', '2'};

/* FNV-1a over the live trie in the order make_automaton numbers it (BFS, children in insertion order): parent's BFS id,
 * edge byte, key id of every node.  Two tries with the same hash flatten to the same tables. */
static uint64_t content_hash(const acb_trie *t) {
    uint64_t h = 1469598103934665603ULL;
    auto mix = [&h](uint64_t v) { for (int i = 0; i < 8; i++) { h ^= (v >> (8 * i)) & 0xff; h *= 1099511628211ULL; } };
    mix((uint64_t)t->letter_bytes);
    if (t->nodes.empty() || t->live_nodes <= 0) return h;
    std::vector<int32_t> order;
    order.reserve((size_t)t->live_nodes);
    order.push_back(0);
    std::vector<int32_t> parent_new;
    parent_new.reserve((size_t)t->live_nodes);
    parent_new.push_back(-1);
    for (size_t i = 0; i < order.size(); i++) {
        const Node &nd = t->nodes[order[i]];
        mix(((uint64_t)(uint32_t)parent_new[i] << 32) | ((uint64_t)nd.byte << 24) | (uint64_t)((uint32_t)nd.key_id & 0xffffffu));
        mix((uint64_t)(uint32_t)nd.key_id);
        for (int32_t c = nd.first_child; c >= 0; c = t->nodes[c].next_sibling)
            if (t->nodes[c].live_below > 0) { order.push_back(c); parent_new.push_back((int32_t)i); }
    }
    return h;
}

template <typename T>
static void put_vec(std::vector<uint8_t> &out, const std::vector<T> &v) {
    const uint64_t n = v.size();
    const uint8_t *p = reinterpret_cast<const uint8_t *>(&n);
    out.insert(out.end(), p, p + 8);
    const uint8_t *d = reinterpret_cast<const uint8_t *>(v.data());
    out.insert(out.end(), d, d + n * sizeof(T));
    while (out.size() % 8) out.push_back(0);
}

template <typename T>
static bool get_vec(const uint8_t *buf, int64_t len, int64_t &pos, std::vector<T> &v, uint64_t max_items) {
    if (pos + 8 > len) return false;
    uint64_t n;
    memcpy(&n, buf + pos, 8);
    pos += 8;
    if (n > max_items || (int64_t)(n * sizeof(T)) > len - pos) return false;
    v.resize((size_t)n);
    if (n) memcpy(v.data(), buf + pos, (size_t)n * sizeof(T));
    pos += (int64_t)(n * sizeof(T));
    pos = (pos + 7) & ~(int64_t)7;
    return pos <= len + 7;
}

struct FlatHeader {
    char magic[8];
    uint64_t hash;
    int32_t abi, letter_bytes, S, K, n_keys, min_key_bytes, max_key_bytes, gram, stride, log1, log3, logA, filter_flags, log2b;
    uint8_t byte_class[256];
};

} // namespace

extern "C" uint64_t acb_trie_content_hash(const acb_trie *t) {
    if (!t) return 0;
    try { return content_hash(t); } catch (const std::exception &) { return 0; }
}

extern "C" int acb_trie_flat_save(const acb_trie *t, uint8_t *out, int64_t cap, int64_t *need) {
    if (!t || !need) { acb_set_error("bad argument"); return ACB_EINVAL; }
    if (t->kind != ACB_AHOCORASICK || !t->flat.valid) { acb_set_error("not an Aho-Corasick automaton yet"); return ACB_ESTATE; }
    try {
        const Flat &f = t->flat;
        std::vector<uint8_t> b;
        FlatHeader h;
        memset(&h, 0, sizeof(h));
        memcpy(h.magic, kFlatMagic, 8);
        h.hash = content_hash(t);
        h.abi = ACB_ABI_VERSION; h.letter_bytes = t->letter_bytes; h.S = f.S; h.K = f.K; h.n_keys = f.n_keys;
        h.min_key_bytes = f.min_key_bytes; h.max_key_bytes = f.max_key_bytes; h.gram = f.gram; h.stride = f.stride;
        h.log1 = f.log1; h.log3 = f.log3; h.logA = f.logA; h.filter_flags = f.filter_flags; h.log2b = f.log2b;
        memcpy(h.byte_class, f.byte_class, 256);
        b.insert(b.end(), reinterpret_cast<uint8_t *>(&h), reinterpret_cast<uint8_t *>(&h) + sizeof(h));
        put_vec(b, f.goto_cm); put_vec(b, f.fail); put_vec(b, f.letter_fail); put_vec(b, f.key_of); put_vec(b, f.out_ptr);
        put_vec(b, f.out_idx); put_vec(b, f.key_len); put_vec(b, f.bm1); put_vec(b, f.bm3); put_vec(b, f.anchors);
        *need = (int64_t)b.size();
        if (out && cap >= (int64_t)b.size()) memcpy(out, b.data(), b.size());
        return ACB_OK;
    } catch (const std::exception &) {
        acb_set_error("out of memory while serialising the flat tables");
        return ACB_ENOMEM;
    }
}

extern "C" int acb_trie_flat_load(acb_trie *t, const uint8_t *buf, int64_t len) {
    if (!t || !buf || len < (int64_t)sizeof(FlatHeader)) { acb_set_error("bad argument"); return ACB_EINVAL; }
    if (t->kind != ACB_TRIE) { acb_set_error("flat tables can only be installed on a trie that has keys and is not built"); return ACB_ESTATE; }
    try {
        FlatHeader h;
        memcpy(&h, buf, sizeof(h));
        if (memcmp(h.magic, kFlatMagic, 8) != 0 || h.abi != ACB_ABI_VERSION || h.letter_bytes != t->letter_bytes ||
            (int64_t)h.S != t->live_nodes || h.hash != content_hash(t)) {
            acb_set_error("flat-table cache does not belong to this key set (or to this library version)");
            return ACB_EINVAL;
        }
        Flat f;
        f.S = h.S; f.K = h.K; f.n_keys = h.n_keys; f.min_key_bytes = h.min_key_bytes; f.max_key_bytes = h.max_key_bytes;
        f.gram = h.gram; f.stride = h.stride; f.log1 = h.log1; f.log3 = h.log3; f.logA = h.logA; f.filter_flags = h.filter_flags; f.log2b = h.log2b;
        memcpy(f.byte_class, h.byte_class, 256);
        int64_t pos = (int64_t)sizeof(FlatHeader);
        const uint64_t big = (uint64_t)1 << 34;
        bool ok = get_vec(buf, len, pos, f.goto_cm, big) && get_vec(buf, len, pos, f.fail, big) && get_vec(buf, len, pos, f.letter_fail, big) &&
                  get_vec(buf, len, pos, f.key_of, big) && get_vec(buf, len, pos, f.out_ptr, big) && get_vec(buf, len, pos, f.out_idx, big) &&
                  get_vec(buf, len, pos, f.key_len, big) && get_vec(buf, len, pos, f.bm1, big) && get_vec(buf, len, pos, f.bm3, big) &&
                  get_vec(buf, len, pos, f.anchors, big);
        ok = ok && f.S > 0 && f.K > 0 && f.K <= 256 && f.goto_cm.size() == (size_t)f.K * f.S && f.fail.size() == (size_t)f.S &&
             f.letter_fail.size() == (size_t)f.S && f.key_of.size() == (size_t)f.S && f.out_ptr.size() == (size_t)f.S + 1 &&
             f.key_len.size() == (size_t)f.n_keys && f.log1 >= 13 && f.log1 <= 20 && ((f.filter_flags & ACB_FILTER_PAIR) ? (f.log2b >= 13 && f.log2b <= 19) : f.log2b == 0) &&
             f.bm1.size() == ((size_t)1 << (f.log1 - 5)) + (f.log2b ? (size_t)1 << (f.log2b - 5) : 0) &&
             f.bm3.size() == (f.log3 ? ((size_t)1 << (f.log3 - 5)) : (size_t)1) && f.logA >= 10 && f.logA <= 28 &&
             f.anchors.size() == ((size_t)8 << f.logA) && !f.out_ptr.empty() && f.out_idx.size() == (size_t)f.out_ptr.back();
        if (!ok) { acb_set_error("flat-table cache is truncated or inconsistent"); return ACB_EINVAL; }
        f.valid = true;
        t->flat = std::move(f);
        t->kind = ACB_AHOCORASICK;
        return ACB_OK;
    } catch (const std::exception &) {
        t->flat = Flat();
        acb_set_error("out of memory while restoring the flat tables");
        return ACB_ENOMEM;
    }
}

/* ------------------------------------------------ the reference's node records (include/acb200.h) */
namespace {

constexpr int kNodeRecBytes = 24;        /* PICKLE_TRIENODE_SIZE on LP64: output 8, fail 8, n 4, eow 1, pad 3 */

static inline void put_u64(uint8_t *p, uint64_t v) { memcpy(p, &v, 8); }
static inline void put_u32(uint8_t *p, uint32_t v) { memcpy(p, &v, 4); }
static inline uint64_t get_u64(const uint8_t *p) { uint64_t v; memcpy(&v, p, 8); return v; }
static inline uint32_t get_u32(const uint8_t *p) { uint32_t v; memcpy(&v, p, 4); return v; }

struct LetterEdge { uint32_t letter; int32_t node; };

/* live letter-children of arena node a: every live node L bytes below it, in the order in which the reference holds
 * them in the node's child array -- the order in which the links were made (Node::birth of the letter's last byte) */
static void letter_children(const acb_trie *t, int32_t a, std::vector<LetterEdge> &out, std::vector<LetterEdge> &tmp) {
    const int L = t->letter_bytes;
    out.clear();
    out.push_back({0u, a});
    for (int d = 0; d < L; d++) {
        tmp.clear();
        for (const LetterEdge &e : out)
            for (int32_t c = t->nodes[e.node].first_child; c >= 0; c = t->nodes[c].next_sibling)
                if (t->nodes[c].live_below > 0) tmp.push_back({e.letter | ((uint32_t)t->nodes[c].byte << (8 * d)), c});
        out.swap(tmp);
    }
    if (out.size() > 1)
        std::sort(out.begin(), out.end(), [t](const LetterEdge &x, const LetterEdge &y) { return t->nodes[x.node].birth < t->nodes[y.node].birth; });
}

/* The walk of the reference's keys() / values() / items(): its iterator keeps a stack, pushes a node's children in array
 * order and pops the last one first (src/AutomatonItemsIter.c:125-288) -- a pre-order walk that takes the youngest
 * child first.  visit(a, tag, kids, kid_tags) sees every live letter node a in that order, with the tag its parent gave
 * it (the root's is 0) and its letter-children oldest first; it sets kid_tags[i], the tag of kids[i]. */
template <typename Visit>
static void key_order_walk(const acb_trie *t, Visit &&visit) {
    std::vector<std::pair<int32_t, int32_t>> stack;
    std::vector<LetterEdge> kids, tmp;
    std::vector<int32_t> tags;
    stack.push_back({0, 0});
    while (!stack.empty()) {
        const auto [a, tag] = stack.back();
        stack.pop_back();
        letter_children(t, a, kids, tmp);
        tags.assign(kids.size(), 0);
        visit(a, tag, kids, tags);
        for (size_t i = 0; i < kids.size(); i++) stack.push_back({kids[i].node, tags[i]});   /* the youngest ends up on top */
    }
}

} // namespace

/* Key ids in the order in which the reference's keys() / values() / items() yield them (key_order_walk). */
extern "C" int acb_trie_key_order(const acb_trie *t, int32_t *out, int64_t cap, int64_t *n) {
    if (!t || !n || cap < 0 || (cap && !out)) { acb_set_error("bad argument"); return ACB_EINVAL; }
    *n = 0;
    if (t->nodes.empty() || t->count == 0) return ACB_OK;
    try {
        int64_t k = 0;
        key_order_walk(t, [&](int32_t a, int32_t, const std::vector<LetterEdge> &, std::vector<int32_t> &) {
            if (t->nodes[a].key_id >= 0) {
                if (k < cap) out[k] = t->nodes[a].key_id;
                k++;
            }
        });
        *n = k;
        if (k > cap) { acb_set_error("key order: room for %lld ids, %lld keys", (long long)cap, (long long)k); return ACB_EOVERFLOW; }
        return ACB_OK;
    } catch (const std::exception &) {
        acb_set_error("out of memory");
        return ACB_ENOMEM;
    }
}

/* The key order as ranges over the flat tables (include/acb200.h).  The same walk as acb_trie_key_order; each letter
 * node's state is found by stepping the flat goto table from its parent's state over the letter's bytes, so the arrays
 * fit the tables also when they came from the flat-table cache. */
extern "C" int acb_trie_key_ranges(const acb_trie *t, int32_t *order, int32_t *lo, int32_t *cnt, int32_t *child_ptr,
                                   int32_t *child, int64_t *n_edges) {
    if (!t || !order || !lo || !cnt || !child_ptr || !child || !n_edges) { acb_set_error("bad argument"); return ACB_EINVAL; }
    if (t->kind != ACB_AHOCORASICK || !t->flat.valid) { acb_set_error("not an Aho-Corasick automaton yet"); return ACB_ESTATE; }
    const Flat &f = t->flat;
    const int L = t->letter_bytes;
    const size_t S = (size_t)f.S;
    *n_edges = 0;
    try {
        std::fill(lo, lo + S, 0);
        std::fill(cnt, cnt + S, 0);
        std::vector<int32_t> deg(S, 0), at(S, 0), kid_states;    /* letter-children of state s: kid_states[at[s] ..][:deg[s]] */
        kid_states.reserve(S);
        int64_t k = 0;
        bool ok = true;
        if (t->count > 0) key_order_walk(t, [&](int32_t a, int32_t s, const std::vector<LetterEdge> &kids, std::vector<int32_t> &tags) {
            const Node &nd = t->nodes[a];
            lo[s] = (int32_t)k;
            cnt[s] = nd.live_below;
            if (nd.key_id >= 0 && k < t->count) order[k++] = nd.key_id;
            at[s] = (int32_t)kid_states.size();
            deg[s] = (int32_t)kids.size();
            for (size_t i = kids.size(); i-- > 0;) {             /* youngest first, the order of the walk: by ascending lo */
                int32_t x = s;
                for (int d = 0; d < L && x >= 0; d++)
                    x = f.goto_cm[(size_t)f.byte_class[(kids[i].letter >> (8 * d)) & 0xffu] * S + (size_t)x];
                if (x <= 0) { ok = false; x = 0; }
                tags[i] = x;
                kid_states.push_back(x);
            }
        });
        if (!ok || k != t->count) { acb_set_error("internal: the flat tables do not fit the trie"); return ACB_EINVAL; }
        child_ptr[0] = 0;
        for (size_t s = 0; s < S; s++) {
            child_ptr[s + 1] = child_ptr[s] + deg[s];
            std::copy(kid_states.begin() + at[s], kid_states.begin() + at[s] + deg[s], child + child_ptr[s]);
        }
        *n_edges = (int64_t)kid_states.size();
        return ACB_OK;
    } catch (const std::exception &) {
        acb_set_error("out of memory");
        return ACB_ENOMEM;
    }
}

extern "C" int acb_trie_export_nodes(const acb_trie *t, int letter_width, const int64_t *value_of_key, int64_t n_values,
                                     uint8_t *out, int64_t cap, int64_t *need_bytes, int64_t *n_nodes,
                                     int64_t *rec_off, int32_t *eow_key, int64_t cap_nodes) {
    if (!t || !need_bytes || !n_nodes) { acb_set_error("bad argument"); return ACB_EINVAL; }
    if (letter_width != (t->letter_bytes == 4 ? 4 : 2)) {          /* TRIE_LETTER_TYPE: u16 (bytes build) or u32, src/common.h:51-67 */
        acb_set_error("letter_width %d does not go with %d-byte letters", letter_width, t->letter_bytes);
        return ACB_EINVAL;
    }
    *need_bytes = 0;
    *n_nodes = 0;
    if (t->nodes.empty() || t->kind == ACB_EMPTY) return ACB_OK;
    try {
        const int L = t->letter_bytes;
        const bool built = (t->kind == ACB_AHOCORASICK) && t->flat.valid;
        /* state numbering of make_automaton (BFS, live nodes, insertion order), to read flat.letter_fail */
        std::vector<int32_t> order, newid;
        if (built) {
            newid.assign(t->nodes.size(), -1);
            order.push_back(0);
            newid[0] = 0;
            for (size_t h = 0; h < order.size(); h++)
                for (int32_t c = t->nodes[order[h]].first_child; c >= 0; c = t->nodes[c].next_sibling)
                    if (t->nodes[c].live_below > 0) { newid[c] = (int32_t)order.size(); order.push_back(c); }
        }
        /* pass 1: pre-order ids (1..N) of the letter nodes */
        std::vector<int32_t> pre;                       /* id-1 -> arena node */
        std::vector<int64_t> id_of(t->nodes.size(), 0); /* arena node -> id, 0 = not a letter node */
        std::vector<LetterEdge> kids, tmp;
        {
            std::vector<int32_t> stack;
            stack.push_back(0);
            while (!stack.empty()) {
                int32_t a = stack.back();
                stack.pop_back();
                pre.push_back(a);
                id_of[a] = (int64_t)pre.size();
                letter_children(t, a, kids, tmp);
                for (size_t i = kids.size(); i-- > 0;) stack.push_back(kids[i].node);   /* first child on top */
            }
        }
        const int64_t N = (int64_t)pre.size();
        const int pair_bytes = letter_width + 8;
        int64_t pos = 0;
        for (int64_t i = 0; i < N; i++) {
            const int32_t a = pre[i];
            letter_children(t, a, kids, tmp);
            const int64_t rec = kNodeRecBytes + (int64_t)kids.size() * pair_bytes;
            if (rec_off && i < cap_nodes) rec_off[i] = pos;
            const int32_t kid = t->nodes[a].key_id;
            if (eow_key && i < cap_nodes) eow_key[i] = kid;
            if (out && pos + rec <= cap) {
                uint8_t *p = out + pos;
                memset(p, 0, (size_t)rec);
                uint64_t output = 0;
                if (kid >= 0 && value_of_key && kid < n_values) output = (uint64_t)value_of_key[kid];
                uint64_t fail = 0;
                if (built && a != 0) {
                    const int32_t lf = t->flat.letter_fail[newid[a]];
                    if (lf >= 0) fail = (uint64_t)id_of[order[lf]];
                }
                put_u64(p, output);
                put_u64(p + 8, fail);
                put_u32(p + 16, (uint32_t)kids.size());
                p[20] = kid >= 0 ? 1 : 0;
                p += kNodeRecBytes;
                for (const LetterEdge &e : kids) {
                    uint32_t letter = e.letter;
                    if (L == 1 && letter_width == 2) letter = (uint32_t)(uint16_t)(int16_t)(int8_t)(uint8_t)letter;   /* src/utils.c:199-202 */
                    memcpy(p, &letter, (size_t)letter_width);
                    put_u64(p + letter_width, (uint64_t)id_of[e.node]);
                    p += pair_bytes;
                }
            }
            pos += rec;
        }
        if (rec_off && N <= cap_nodes) rec_off[N] = pos;            /* rec_off has cap_nodes + 1 slots */
        *need_bytes = pos;
        *n_nodes = N;
        if (out && pos > cap) { acb_set_error("export buffer too small: %lld > %lld", (long long)pos, (long long)cap); return ACB_EOVERFLOW; }
        if ((rec_off || eow_key) && N > cap_nodes) { acb_set_error("node arrays too small"); return ACB_EOVERFLOW; }
        return ACB_OK;
    } catch (const std::bad_alloc &) {
        acb_set_error("out of memory");
        return ACB_ENOMEM;
    } catch (const std::exception &e) {                      /* e.g. std::length_error: nothing may cross the C ABI */
        acb_set_error("%s", e.what());
        return ACB_EINVAL;
    }
}

extern "C" int acb_trie_import_nodes(acb_trie *t, const uint8_t *buf, int64_t len, int64_t n_nodes, int letter_width, int mode,
                                     int store_any, int64_t *out_value, int64_t *out_blob_off, int64_t cap_keys, int64_t *n_keys,
                                     int64_t *consumed, uint8_t *key_bytes, int64_t key_cap, int64_t *key_off, int64_t *key_need) {
    if (!t || !n_keys || len < 0 || n_nodes < 0 || (len && !buf)) { acb_set_error("bad argument"); return ACB_EINVAL; }
    if (letter_width != (t->letter_bytes == 4 ? 4 : 2)) { acb_set_error("letter_width %d does not go with %d-byte letters", letter_width, t->letter_bytes); return ACB_EINVAL; }
    if (mode != ACB_NODES_PICKLE && mode != ACB_NODES_SAVE) { acb_set_error("unknown record mode %d", mode); return ACB_EINVAL; }
    if (!t->nodes.empty()) { acb_set_error("import needs an empty trie"); return ACB_EINVAL; }
    *n_keys = 0;
    if (consumed) *consumed = 0;
    if (key_need) *key_need = 0;
    if (key_off && cap_keys >= 0) key_off[0] = 0;
    if (n_nodes == 0) return ACB_OK;
    if (n_nodes > len / (kNodeRecBytes + (mode == ACB_NODES_SAVE ? 8 : 0))) {     /* before anything is sized by it */
        acb_set_error("%lld nodes announced, but the data can hold at most %lld", (long long)n_nodes,
                      (long long)(len / (kNodeRecBytes + (mode == ACB_NODES_SAVE ? 8 : 0))));
        return ACB_EINVAL;
    }
    try {
        const int L = t->letter_bytes;
        const int pair_bytes = letter_width + 8;
        /* pass 1: locate the records */
        std::vector<int64_t> rec(n_nodes), blob(n_nodes, -1);
        std::vector<std::pair<uint64_t, int64_t>> by_addr;          /* SAVE: address -> node index */
        if (mode == ACB_NODES_SAVE) by_addr.reserve(n_nodes);
        int64_t pos = 0;
        for (int64_t i = 0; i < n_nodes; i++) {
            if (mode == ACB_NODES_SAVE) {
                if (pos + 8 > len) { acb_set_error("truncated: address of node %lld", (long long)i); return ACB_EINVAL; }
                by_addr.emplace_back(get_u64(buf + pos), i);
                pos += 8;
            }
            if (pos + kNodeRecBytes > len) { acb_set_error("truncated: header of node %lld", (long long)i); return ACB_EINVAL; }
            rec[i] = pos;
            const uint64_t n = get_u32(buf + pos + 16);
            const bool eow = buf[pos + 20] != 0;
            const uint64_t output = get_u64(buf + pos);
            pos += kNodeRecBytes;
            if (n > (uint64_t)(len - pos) / (uint64_t)pair_bytes) { acb_set_error("truncated: children of node %lld", (long long)i); return ACB_EINVAL; }
            pos += (int64_t)n * pair_bytes;
            if (mode == ACB_NODES_SAVE && store_any && eow) {
                if (output > (uint64_t)(len - pos)) { acb_set_error("truncated: value of node %lld", (long long)i); return ACB_EINVAL; }
                blob[i] = pos;
                pos += (int64_t)output;
            }
        }
        if (consumed) *consumed = pos;
        if (mode == ACB_NODES_SAVE) {
            std::sort(by_addr.begin(), by_addr.end());
            for (size_t i = 1; i < by_addr.size(); i++)
                if (by_addr[i].first == by_addr[i - 1].first) { acb_set_error("two nodes share one address"); return ACB_EINVAL; }
        }
        auto resolve = [&](uint64_t ref) -> int64_t {
            if (mode == ACB_NODES_PICKLE) return (ref >= 1 && ref <= (uint64_t)n_nodes) ? (int64_t)ref - 1 : -1;
            auto it = std::lower_bound(by_addr.begin(), by_addr.end(), std::make_pair(ref, (int64_t)-1));
            return (it != by_addr.end() && it->first == ref) ? it->second : -1;
        };
        /* pass 2: pre-order walk from the first record (the root), entering the keys */
        struct Frame { int64_t node; uint32_t next_child; };
        std::vector<Frame> stack;
        std::vector<uint8_t> path;
        std::vector<uint8_t> seen(n_nodes, 0);
        stack.push_back({0, 0});
        seen[0] = 1;
        int64_t keys = 0, kbytes = 0;
        auto visit = [&](int64_t i) -> int {
            const uint8_t *p = buf + rec[i];
            if (p[20]) {                                   /* eow */
                if (path.empty()) { acb_set_error("the root is marked as the end of a key"); return ACB_EINVAL; }
                if (keys >= 0x7fffffff) { acb_set_error("too many keys"); return ACB_ERANGE; }
                if (keys < cap_keys) {
                    if (out_value) out_value[keys] = (int64_t)get_u64(p);
                    if (out_blob_off) out_blob_off[keys] = blob[i];
                    if (key_bytes && key_off && kbytes + (int64_t)path.size() <= key_cap) {
                        memcpy(key_bytes + kbytes, path.data(), path.size());
                        key_off[keys + 1] = kbytes + (int64_t)path.size();
                    }
                }
                kbytes += (int64_t)path.size();
                int rc = acb_trie_add_word(t, path.data(), (int64_t)path.size(), (int32_t)keys, nullptr);
                if (rc != ACB_OK) return rc;
                keys++;
            }
            return ACB_OK;
        };
        while (!stack.empty()) {
            Frame &f = stack.back();
            const uint8_t *p = buf + rec[f.node];
            const uint32_t n = get_u32(p + 16);
            if (f.next_child == n) {
                stack.pop_back();
                if (!stack.empty()) path.resize(path.size() - L);
                continue;
            }
            const uint8_t *pr = p + kNodeRecBytes + (size_t)f.next_child * pair_bytes;
            f.next_child++;
            uint32_t letter = 0;
            memcpy(&letter, pr, (size_t)letter_width);
            const int64_t child = resolve(get_u64(pr + letter_width));
            if (child < 0) { acb_set_error("node %lld: child link does not point to a node", (long long)f.node); return ACB_EINVAL; }
            if (seen[child]) { acb_set_error("node %lld is reachable twice", (long long)child); return ACB_EINVAL; }
            seen[child] = 1;
            if (L == 1) {
                if (letter > 0xffu && letter < 0xff80u) { acb_set_error("letter %u does not fit a byte", letter); return ACB_EINVAL; }
                path.push_back((uint8_t)(letter & 0xffu));           /* undo the sign extension */
            } else if (L == 2) {
                if (letter > 0xffffu) { acb_set_error("letter %u does not fit 16 bits", letter); return ACB_EINVAL; }
                path.push_back((uint8_t)(letter & 0xff)); path.push_back((uint8_t)(letter >> 8));
            } else {
                for (int b = 0; b < 4; b++) path.push_back((uint8_t)(letter >> (8 * b)));
            }
            stack.push_back({child, 0});                 /* invalidates f */
            int rc = visit(child);
            if (rc != ACB_OK) return rc;
        }
        *n_keys = keys;
        if (key_need) *key_need = kbytes;
        if (keys > cap_keys && (out_value || out_blob_off || key_off)) { acb_set_error("key arrays too small"); return ACB_EOVERFLOW; }
        if (key_bytes && kbytes > key_cap) { acb_set_error("key byte buffer too small"); return ACB_EOVERFLOW; }
        return ACB_OK;
    } catch (const std::bad_alloc &) {
        acb_set_error("out of memory");
        return ACB_ENOMEM;
    } catch (const std::exception &e) {                      /* e.g. std::length_error: nothing may cross the C ABI */
        acb_set_error("%s", e.what());
        return ACB_EINVAL;
    }
}

extern "C" int acb_node_records_span(const uint8_t *buf, int64_t len, int64_t n_nodes, int letter_width, int64_t *span) {
    if (!span || len < 0 || n_nodes < 0 || (len && !buf) || (letter_width != 2 && letter_width != 4)) { acb_set_error("bad argument"); return ACB_EINVAL; }
    const int pair_bytes = letter_width + 8;
    int64_t pos = 0;
    for (int64_t i = 0; i < n_nodes; i++) {
        if (pos + kNodeRecBytes > len) { acb_set_error("Data truncated [parsing header of node #%lld]", (long long)i); return ACB_EINVAL; }
        const uint64_t n = get_u32(buf + pos + 16);
        pos += kNodeRecBytes;
        if (n > (uint64_t)(len - pos) / (uint64_t)pair_bytes) { acb_set_error("Data truncated [parsing children of node #%lld]", (long long)i); return ACB_EINVAL; }
        pos += (int64_t)n * pair_bytes;
    }
    *span = pos;
    return ACB_OK;
}

/* ------------------------------------------------------------- white space */
/* The letters iter(..., ignore_white_space=True) skips (src/AutomatonSearchIter.c:270-274): libc iswspace() under the
 * current LC_CTYPE, of the letter as the reference widens it (src/utils.c:199-202 for the bytes build). */
extern "C" int acb_space_letters(int letter_bytes, int signed_bytes, uint32_t *out, int64_t cap, int64_t *n) {
    if (!n || cap < 0 || (cap && !out) || (letter_bytes != 1 && letter_bytes != 2 && letter_bytes != 4)) { acb_set_error("bad argument"); return ACB_EINVAL; }
    const uint32_t last = letter_bytes == 1 ? 0xffu : (letter_bytes == 2 ? 0xffffu : 0x10ffffu);   /* no code point past U+10FFFF */
    int64_t k = 0;
    for (uint32_t v = 0; v <= last; v++) {
        const uint32_t w = (letter_bytes == 1 && signed_bytes) ? (uint32_t)(uint16_t)(int16_t)(int8_t)(uint8_t)v : v;
        if (!iswspace((wint_t)w)) continue;
        if (k < cap) out[k] = v;
        k++;
    }
    *n = k;
    if (k > cap) { acb_set_error("%lld white-space letters, capacity %lld", (long long)k, (long long)cap); return ACB_EOVERFLOW; }
    return ACB_OK;
}
