/*
 * acb_device.cu -- sm_90a scan kernels and the device half of the C ABI (include/acb200.h).
 *
 * ACB_ALGO_FILTER (the fast path) is ONE launch per <= 2 GiB segment of the batch, of one of two streaming kernels
 * (both persistent, one CTA per SM, warp specialised):
 *
 *  acb_stream_kernel<NW,STRIDE,MODE>   SINGLE placements of the gram filter (any gram length and stride)
 *  acb_pair_kernel<L2B>                PAIR placement (gram 4, stride 1, 1-byte letters: one filter word per two positions)
 *      A producer warp claims tiles of the flat haystack buffer from an atomic counter (20 KiB into a 3-stage ring;
 *      pair kernel: 32 KiB into 2 stages) and moves them into shared memory with cp.async.bulk (the TMA engine) and
 *      mbarriers; the consumer warps take
 *      1 KiB slices of the stages from a shared-memory counter, hash the gram at every probe position and test it
 *      against the gram bitmap held in shared memory.  Start-anchored search: the rare survivors get the second
 *      hash of their gram (read back from the stage, still resident) and are collected per warp; a warp that has 32 of
 *      them resolves them through the anchor table in global memory (one 32-byte slot): a UNIQUE anchor carries the
 *      only key that can match there, which is compared with the text directly; a MULTI anchor (keys sharing that
 *      prefix) walks the trie through the column-major goto table.  No failure links are followed: an occurrence is
 *      found exactly once, from its first byte, so the result set equals what the reference produces by walking fail
 *      chains at every position (src/AutomatonSearchIter.c:157-197, src/Automaton.c:693-714).
 *
 *  acb_dfa_kernel                      (ACB_ALGO_DFA)
 *      The textbook automaton: goto, else fail until root (src/trie.c:177-194), outputs from CSR lists.  One
 *      lane per 64-byte span with a max_key-1 byte warm-up.  Slower (every byte is a dependent L2 lookup) but
 *      insensitive to key-set shape; also used to cross-check the stream kernel on the GPU.
 *
 *  acb_long_kernel                     (ACB_ALGO_LONG)
 *      iter_long: the reference's longest-match walk (src/AutomatonSearchIterLong.c:89-153) replayed letter by
 *      letter on the flattened tables, one lane per haystack.
 *
 * Match records are appended to the global buffer with one atomicAdd per warp flush (stream kernel: staged in shared
 * memory) or per resolve turn (pair kernel); acb_sort_matches_device puts them into the reference's order with one radix sort.
 */
#include "acb_internal.h"
#include "acb_hash.h"

#include <cuda_runtime.h>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>

#include <algorithm>
#include <atomic>
#include <cassert>
#include <mutex>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <exception>
#include <new>
#include <type_traits>
#include <vector>

#define CUDA_TRY(expr)                                                                       \
    do {                                                                                     \
        cudaError_t _e = (expr);                                                             \
        if (_e != cudaSuccess) {                                                             \
            acb_set_error("CUDA error %s at %s:%d: %s", cudaGetErrorName(_e), __FILE__,      \
                          __LINE__, cudaGetErrorString(_e));                                 \
            return ACB_ECUDA;                                                                \
        }                                                                                    \
    } while (0)

namespace {

#ifndef ACB_CONSUMERS
#define ACB_CONSUMERS 31
#endif
#ifndef ACB_STAGES
#define ACB_STAGES 3
#endif
#ifndef ACB_LANE_BYTES
#define ACB_LANE_BYTES 32
#endif
constexpr int kConsumers    = ACB_CONSUMERS;          /* consumer warps of the stream kernel           */
constexpr int kFThreads     = (kConsumers + 1) * 32;  /* + the producer warp                           */
constexpr int kLaneBytes    = ACB_LANE_BYTES;         /* text bytes per lane and iteration             */
constexpr int kLaneWords    = kLaneBytes / 4;
constexpr int kSliceBytes   = 32 * kLaneBytes;        /* one warp iteration                            */
#ifndef ACB_TILE_SLICES
#define ACB_TILE_SLICES 20
#endif
constexpr int kTileSlices   = ACB_TILE_SLICES;        /* slices per tile (= arrivals on a stage's empty barrier).  Slices are handed out in order,
                                                         one per warp at a time, so the fills in use span at most kConsumers / kTileSlices + 2
                                                         consecutive ones: less than 2 * kStages, and no barrier phase can alias */
constexpr int kTileBytes    = kTileSlices * kSliceBytes;
constexpr int kLook         = 16;                     /* bytes copied past a tile (gram look-ahead)    */
constexpr int kStageBytes   = (kTileBytes + kLook + 127) / 128 * 128;   /* tile + look-ahead, stages stay 128 B aligned */
constexpr int kStages       = ACB_STAGES;
constexpr int kClaimDepth   = 8;                      /* tile claims in flight per producer            */
constexpr int kWarpCand     = kSliceBytes + 32;       /* candidate entries per consumer warp: a warp resolves them as soon as it
                                                         has 32, and one slice adds at most kSliceBytes (one per byte) */
constexpr int kStageCap     = 64;                     /* match records staged per consumer warp (smem) */
static_assert((kConsumers + kTileSlices - 1) / kTileSlices + 2 < 2 * ACB_STAGES, "ring too shallow for the slice hand-out");
static_assert(kFThreads <= 1024 && kTileBytes % 16 == 0 && kLaneBytes == 32 && kStageCap * 12 / 2 >= 8 * 32, "stream kernel shape");
constexpr uint32_t kFull    = 0xffffffffu;
constexpr uint32_t kNoTile  = 0xffffffffu;
constexpr int32_t  kTermBit = 0x40000000;             /* goto entry flag: child ends a key             */
constexpr int32_t  kIdMask  = 0x3fffffff;
constexpr long long kSegBytes = 1LL << 31;            /* candidates are uint32 offsets into a segment  */

constexpr int kDfaSpan      = 64;                     /* bytes per lane in the DFA kernel              */
constexpr int kDfaThreads   = 256;

enum { kModeNarrow = 0, kModeWide = 1 };                  /* how a SINGLE gram is placed in the bitmap (acb_hash.h); PAIR has its own kernel */

std::atomic<long long> g_launches{0};
thread_local float g_last_ms = 0.f;
thread_local float g_compact_ms = 0.f, g_remap_ms = 0.f;   /* kernel timing of the last white-space scan */
std::atomic<int> g_timing{0};

struct ScanParams {
    const uint8_t *hay;
    long long total;
    const long long *offsets;      /* nullptr => fixed stride */
    long long n_hay;
    long long stride_bytes;
    const uint8_t *cls;
    const int32_t *gto;            /* flagged goto (kTermBit) */
    const int32_t *fail;
    const int32_t *letter_fail;
    const int32_t *key_of;
    const int32_t *out_ptr;
    const int32_t *out_idx;
    const int32_t *key_len;
    int32_t S;
    int32_t L;
    int32_t gram;
    int32_t max_key_bytes;
    const uint32_t *bm1;           /* gram bitmap, 2^(log1-5) words */
    const uint32_t *bm3;           /* tag bitmap in global memory, 2^log3 bits; log3 == 0: not built */
    const uint4 *anchors;          /* 2 x uint4 per slot */
    int32_t log1, log3, logA;
    int32_t log2b;                 /* PAIR: level 2 (behind level 1 in bm1) has 2^log2b bits */
    uint32_t mul1[ACB_MAX_WINDOWS];
    uint32_t mul2[ACB_MAX_WINDOWS];
    acb_match *out;
    long long cap;
    unsigned long long *count;
    int32_t long_init;             /* ACB_ALGO_LONG: the state haystack 0 starts in (iter_long streaming) */
    int32_t *long_final;           /* ... and where the state it ends in goes (may be null) */
    long long seg_begin, seg_end;  /* byte range of this launch */
    unsigned int n_tiles;          /* tiles in the segment (kTileBytes, pair kernel: kPairTileBytes) */
    unsigned int *work_ctr;        /* [0] next tile, [1] CTAs done */
    uint2 *cand;                   /* candidate entries, kWarpCand per consumer warp of every CTA: {position in the segment, anchor tag} */
    int stride_shift;              /* log2(stride_bytes) when it is a power of two, else -1 */
    int letter_shift;              /* log2(L) */
    const int32_t *long_start;     /* ACB_ALGO_LONG of a stream batch: the state every haystack starts in (nullptr: long_init / root) */
    int32_t *long_end;             /* ... and where the state every haystack ends in goes (may be null) */
};

/* ---------------------------------------------------------------- helpers */

/* aligned 32-bit word at byte offset a (a % 4 == 0), zero filled past the end of the buffer */
__device__ __forceinline__ uint32_t load_word(const uint8_t *hay, long long a, long long total) {
    if (a + 4 <= total) return __ldg(reinterpret_cast<const uint32_t *>(hay + a));
    uint32_t v = 0;
    for (int b = 0; b < 4; b++) if (a + b < total) v |= (uint32_t)hay[a + b] << (8 * b);
    return v;
}

/* P: ScanParams, or the pair kernel's PairTurnArgs (the same fields, held in shared memory) */
template <class P>
__device__ __forceinline__ void find_haystack(const P &p, long long q, long long &h, long long &hs, long long &he) {
    if (p.offsets == nullptr) {
        if (p.stride_shift >= 0) h = q >> p.stride_shift;
        else if (p.total <= 0xffffffffLL) h = (long long)((uint32_t)q / (uint32_t)p.stride_bytes);
        else h = q / p.stride_bytes;
        hs = h * p.stride_bytes;
        he = hs + p.stride_bytes;
    } else {
        long long lo = 0, hi = p.n_hay;       /* largest h with offsets[h] <= q */
        while (hi - lo > 1) {
            long long mid = (lo + hi) >> 1;
            if (__ldg(p.offsets + mid) <= q) lo = mid; else hi = mid;
        }
        h = lo;
        hs = __ldg(p.offsets + lo);
        he = __ldg(p.offsets + lo + 1);
    }
}

struct WarpStage {            /* per-warp match staging in shared memory */
    acb_match *buf;
    int *cnt;
};

__device__ __forceinline__ void emit(const ScanParams &p, const WarpStage &ws, int32_t h, int32_t e, int32_t k) {
    acb_match m;
    m.hay_id = h;
    m.end_index = e;
    m.key_id = k;
    int slot;                                 /* ws.cnt is shared memory: a shared-space atomic, not a generic one */
    asm volatile("atom.shared.add.u32 %0, [%1], 1;" : "=r"(slot) : "r"((uint32_t)__cvta_generic_to_shared(ws.cnt)) : "memory");
    if (slot < kStageCap) {
        ws.buf[slot] = m;
    } else {                                  /* staging full: straight to global */
        unsigned long long g = atomicAdd(p.count, 1ULL);
        if (g < (unsigned long long)p.cap) p.out[g] = m;
    }
}

/* all 32 lanes must call; flushes the staged records with one global atomic */
__device__ __forceinline__ void flush_stage(const ScanParams &p, const WarpStage &ws, int lane) {
    __syncwarp();
    int n = *ws.cnt;
    if (n > kStageCap) n = kStageCap;
    if (n > 0) {
        unsigned long long base = 0;
        if (lane == 0) base = atomicAdd(p.count, (unsigned long long)n);
        base = __shfl_sync(kFull, base, 0);
#pragma unroll
        for (int i = lane; i < kStageCap; i += 32)
            if (i < n && base + i < (unsigned long long)p.cap) p.out[base + i] = ws.buf[i];
    }
    __syncwarp();
    if (lane == 0) *ws.cnt = 0;
    __syncwarp();
}

/* stage 3 (MULTI anchors only): walk the trie from the root at `start` */
__device__ __forceinline__ void walk_from(const ScanParams &p, const WarpStage &ws, long long start,
                                          long long h, long long hs, long long he) {
    const int L = p.L;
    int32_t st = 0;
    for (long long i = start; i < he; ++i) {
        int c = __ldg(p.cls + p.hay[i]);
        int32_t nx = __ldg(p.gto + (long long)c * p.S + st);
        if (nx < 0) break;
        st = nx & kIdMask;
        if (nx & kTermBit) {
            int32_t k = __ldg(p.key_of + st);
            emit(p, ws, (int32_t)h, (int32_t)((i - hs + 1) / L - 1), k);
        }
    }
}

/* six aligned words covering the 20 text bytes from x on (zero fill past the end of the buffer) */
template <class P>
__device__ __forceinline__ void load_text(const P &p, long long x, uint32_t (&w)[6]) {
    const long long x0 = x & ~3LL;
    if (x0 + 24 <= p.total) {
        const uint32_t *a = reinterpret_cast<const uint32_t *>(p.hay + x0);
#pragma unroll
        for (int i = 0; i < 6; i++) w[i] = __ldg(a + i);
    } else {
#pragma unroll
        for (int i = 0; i < 6; i++) w[i] = load_word(p.hay, x0 + 4 * i, p.total);
    }
}

/* do the n (<= 20) text bytes at x (words w = load_text(x)) equal the packed bytes kw? */
__device__ __forceinline__ bool text_equals(const uint32_t (&w)[6], long long x, int n, const uint32_t kw[5]) {
    const int sh = (int)(x & 3) * 8;
    uint32_t diff = 0;
#pragma unroll
    for (int i = 0; i < 5; i++) {
        uint32_t t = __funnelshift_r(w[i], w[i + 1], sh);
        int nb = n - 4 * i;                                   /* bytes of this word that count */
        uint32_t mask = nb >= 4 ? 0xffffffffu : (nb <= 0 ? 0u : ((1u << (8 * nb)) - 1u));
        diff |= (t ^ kw[i]) & mask;
    }
    return diff == 0;
}

/* ------------------------------------------------------- the stream kernel */

__device__ __forceinline__ unsigned long long mul_wide(uint32_t a, uint32_t b) {
    unsigned long long d;
    asm("mul.wide.u32 %0, %1, %2;" : "=l"(d) : "r"(a), "r"(b));
    return d;
}
__device__ __forceinline__ unsigned long long mad_wide(uint32_t a, uint32_t b, unsigned long long c) {
    unsigned long long d;
    asm("mad.wide.u32 %0, %1, %2, %3;" : "=l"(d) : "r"(a), "r"(b), "l"(c));
    return d;
}
__device__ __forceinline__ uint32_t lds32(uint32_t saddr) {
    uint32_t v;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(saddr));
    return v;
}
__device__ __forceinline__ uint2 lds64(uint32_t saddr) {
    uint2 v;
    asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(saddr) : "memory");
    return v;
}
__device__ __forceinline__ uint32_t lds16(uint32_t saddr) {
    uint32_t v;
    asm volatile("{ .reg .u16 h; ld.shared.u16 h, [%1]; cvt.u32.u16 %0, h; }" : "=r"(v) : "r"(saddr) : "memory");
    return v;
}
__device__ __forceinline__ void sts16(uint32_t saddr, uint32_t v) {
    asm volatile("{ .reg .u16 h; cvt.u16.u32 h, %1; st.shared.u16 [%0], h; }" :: "r"(saddr), "r"(v) : "memory");
}
__device__ __forceinline__ uint4 lds128(uint32_t saddr) {
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(saddr));
    return v;
}
/* the bitmap never changes during a launch: a plain (non-volatile) load the compiler may schedule freely */
__device__ __forceinline__ uint32_t lds_bitmap(uint32_t saddr) {
    uint32_t v;
    asm("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(saddr));
    return v;
}

/* mbarrier / bulk-copy (TMA engine) primitives: PTX ISA "mbarrier", "cp.async.bulk" */
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred P1;\n"
        "LAB_WAIT:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
        "@P1 bra DONE;\n"
        "bra LAB_WAIT;\n"
        "DONE:\n"
        "}" :: "r"(bar), "r"(parity) : "memory");
}
/* global -> shared bulk copy, completion counted in bytes on `bar`; all of dst, src, bytes are multiples of 16 */
__device__ __forceinline__ void bulk_load(uint32_t dst, const void *src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 :: "r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}

/* Follow the anchor chain of `tag` for the candidate at q, starting with the slot (e0, e1) already loaded.
 * Three ways out, in the order of their frequency on sparse-match text: an empty slot (the bitmap let a foreign
 * gram through); ONE entry that is the last of its tag, UNIQUE and anchored at its first byte (every such lane of
 * the warp runs the same straight-line compare); anything else takes the general loop. */
__device__ __forceinline__ void resolve_chain(const ScanParams &p, const WarpStage &ws, long long q, uint32_t tag,
                                              const uint32_t (&tq)[6], uint4 e0, uint4 e1) {
    if (e0.x == 0u) return;
    long long h = -1, hs = 0, he = 0;
    if (e0.x == tag && (int32_t)e0.y >= 0 && (e0.z & 0x100ffu) == 0x10000u) {
        const uint32_t kw[5] = {e0.w, e1.x, e1.y, e1.z, e1.w};
        const int len = (int)((e0.z >> 8) & 0xffu);
        find_haystack(p, q, h, hs, he);
        if (q + len <= he && text_equals(tq, q, len, kw))
            emit(p, ws, (int32_t)h, (int32_t)(((q + len - hs) >> p.letter_shift) - 1), (int32_t)e0.y);
        return;
    }
    const uint32_t amask = (1u << p.logA) - 1u;
    uint32_t slot = tag >> (32 - p.logA);
    for (;;) {
        if (e0.x == 0u) break;                                 /* empty slot ends the probe sequence */
        if (e0.x == tag) {
            const uint32_t kw[5] = {e0.w, e1.x, e1.y, e1.z, e1.w};
            const int j = (int)(e0.z & 0xffu), len = (int)((e0.z >> 8) & 0xffu);
            const int32_t kid = (int32_t)e0.y;
            if (h < 0) find_haystack(p, q, h, hs, he);
            const long long start = q - j;
            if (start >= hs) {
                if (kid >= 0) {                                /* UNIQUE: the only key that can match at start */
                    bool eq = false;
                    if (start + len <= he) {
                        if (j == 0) eq = text_equals(tq, q, len, kw);
                        else { uint32_t ts[6]; load_text(p, start, ts); eq = text_equals(ts, start, len, kw); }
                    }
                    if (eq) emit(p, ws, (int32_t)h, (int32_t)(((start + len - hs) >> p.letter_shift) - 1), kid);
                } else if (q + len <= he && text_equals(tq, q, len, kw)) {   /* MULTI: exact gram, then the trie */
                    walk_from(p, ws, start, h, hs, he);
                }
            }
            if (e0.z & 0x10000u) break;                        /* no further entry carries this tag */
        }
        slot = (slot + 1) & amask;
        e0 = __ldg(p.anchors + 2 * (size_t)slot);
        e1 = __ldg(p.anchors + 2 * (size_t)slot + 1);
    }
}

/* what a consumer warp needs to probe a slice */
struct ProbeCtx {
    uint32_t sbm;              /* shared-memory address of the bitmap */
    uint32_t n_words;          /* umulhi(h, n_words) = word index */
    uint32_t four;             /* == 4, opaque to the compiler so the address is one IMAD (FMA pipe, which has room) */
    uint32_t two;              /* == 2, same trick for the hit accumulator */
    int sh_bit;                /* NARROW: h >> sh_bit supplies the first bit index (low 5 bits, wrap shift); */
};

/* window t of the lane's text: the 4 bytes at byte offset t of W[] (little endian) */
template <int N>
__device__ __forceinline__ uint32_t window(const uint32_t (&W)[N], int t) {
    return ((t & 3) == 0) ? W[t >> 2] : __funnelshift_r(W[t >> 2], W[(t >> 2) + 1], (t & 3) * 8);
}

/* One bitmap probe per STRIDE-th position of the lane's kLaneBytes bytes; returns bit i = probe i passed.  The hit
 * bit is shifted into `acc` with a multiply-add (FMA pipe; c.two == 2 is opaque to the compiler).  Blocked Bloom,
 * k = 2: both bits of the gram must be set in its word (wrap shifts use the low 5 bits of their amount).
 * WIDE (g % 4 == 0): 64-bit products, low half = hash1 (word index, second bit), high half -> first bit. */
template <int NW, int STRIDE, bool WIDE>
__device__ __forceinline__ uint32_t probe_single(const ProbeCtx &c, const uint32_t (&W)[kLaneWords + NW], const uint32_t (&mul)[NW]) {
    constexpr int kProbes = kLaneBytes / STRIDE;
    uint32_t acc = 0;
#pragma unroll
    for (int t = 0; t < kLaneBytes; t += STRIDE) {
        uint32_t h = 0, ha;
        if (WIDE) {
            unsigned long long hw = 0;
#pragma unroll
            for (int k = 0; k < NW; k++) hw = mad_wide(window(W, t + 4 * k), mul[k], hw);
            h = (uint32_t)hw;
            ha = (uint32_t)(hw >> 32);
        } else {
#pragma unroll
            for (int k = 0; k < NW; k++) h += window(W, t + 4 * k) * mul[k];
            ha = h >> c.sh_bit;
        }
        const uint32_t word = lds_bitmap(__umulhi(h, c.n_words) * c.four + c.sbm);
        const uint32_t both = __funnelshift_r(word, 0u, ha) & __funnelshift_r(word, 0u, h) & 1u;
        acc = acc * c.two + both;
    }
    return __brev(acc) >> (32 - kProbes);
}

/* shared-memory carve-up of the stream kernel (host and device agree through this one function) */
struct StreamSmem {
    uint32_t bitmap, stages, stage_rec, stage_cnt, bars, tiles, next, total;
};
__host__ __device__ inline StreamSmem stream_smem(int log1) {
    StreamSmem s;
    uint32_t o = 0;
    s.bitmap = o;    o += 1u << (log1 - 3);                       o = (o + 127u) & ~127u;
    s.stages = o;    o += (uint32_t)kStages * kStageBytes;
    s.stage_rec = o; o += (uint32_t)kConsumers * kStageCap * (uint32_t)sizeof(acb_match);
    s.stage_cnt = o; o += (uint32_t)kConsumers * 4u;              o = (o + 15u) & ~15u;
    s.bars = o;      o += 2u * kStages * 8u;                      /* full[kStages], empty[kStages] */
    s.tiles = o;     o += (uint32_t)kStages * 4u;
    s.next = o;      o += 4u;                                     /* next slice to hand out */
    s.total = (o + 15u) & ~15u;
    return s;
}

/* A consumer warp's collected candidates {position in the segment, tag}, entries [0, n) of its list, through the anchor
 * table: one entry per lane and turn, the text at the position and the anchor slot its tag hashes to loaded together
 * (one round trip; a second entry per lane makes ptxas spill inside the probe loop).  Text and anchors come from L2:
 * the bytes were streamed microseconds ago.  Records are flushed when the staging area is a quarter full. */
__device__ __forceinline__ void resolve_backlog(const ScanParams &p, uint8_t *smem_raw, unsigned int n) {
    /* everything but n is rebuilt here rather than kept alive across the probe loop */
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const StreamSmem lay = stream_smem(p.log1);
    WarpStage ws;
    ws.buf = reinterpret_cast<acb_match *>(smem_raw + lay.stage_rec) + warp * kStageCap;
    ws.cnt = reinterpret_cast<int *>(smem_raw + lay.stage_cnt) + warp;
    const uint2 *list = p.cand + ((size_t)blockIdx.x * kConsumers + warp) * kWarpCand;
    __syncwarp();                                                        /* the entries were written by other lanes of this warp */
    for (unsigned int i0 = 0; i0 < n; i0 += 32) {
        const unsigned int i = i0 + lane;
        if (i < n) {
            const uint2 e = __ldcg(list + i);
            const long long q = p.seg_begin + (long long)e.x;
            uint32_t tq[6];
            load_text(p, q, tq);
            const uint32_t slot = e.y >> (32 - p.logA);
            const uint4 a0 = __ldg(p.anchors + 2 * (size_t)slot), a1 = __ldg(p.anchors + 2 * (size_t)slot + 1);
            resolve_chain(p, ws, q, e.y, tq, a0, a1);
        }
        __syncwarp();
        if (*reinterpret_cast<volatile int *>(ws.cnt) >= kStageCap / 4) flush_stage(p, ws, lane);    /* warp-uniform */
    }
    flush_stage(p, ws, lane);
}

/* The producer warp of a streaming kernel: claims tiles from the global counter and keeps the shared-memory ring full
 * (cp.async.bulk + mbarrier); `stages` = offset of the ring in the CTA's shared memory.  The ring's geometry (TSLICES
 * slices per tile, STAGES stages) is the kernel's: the pair kernel has its own. */
template <int NCONS, int TSLICES, int STAGES>
__device__ __forceinline__ void stream_producer(const ScanParams &p, uint8_t *smem_raw, uint32_t sbase, uint32_t stages,
                                                uint32_t bar_full, uint32_t bar_empty, volatile uint32_t *s_tile, int lane) {
    constexpr int kTileSlices = TSLICES, kStages = STAGES;
    constexpr int kTileBytes = kTileSlices * kSliceBytes;
    constexpr int kStageBytes = (kTileBytes + kLook + 127) / 128 * 128;
    struct { uint32_t stages; } lay = {stages};
        /* ---------------- producer warp.  Tiles come from one global counter.  A claim is a ~1 us round trip to L2, so
       kClaimDepth of them are kept in flight: claim[k] serves fills k, k + kClaimDepth, ... and is re-issued as soon
       as it has been read (one register per slot, so that reading a slot never waits for a younger atomic). */
    const uint8_t *seg = p.hay + p.seg_begin;
    const long long exist = p.total - p.seg_begin;                   /* bytes that exist from seg onwards */
    unsigned int claim[kClaimDepth];
#pragma unroll
    for (int k = 0; k < kClaimDepth; k++) claim[k] = (lane == 0) ? atomicAdd(p.work_ctr, 1u) : 0u;
    bool more = true;
    for (uint32_t base = 0; more; base += kClaimDepth) {
#pragma unroll
        for (int k = 0; k < kClaimDepth; k++) {
            if (!more) break;
            const uint32_t fill = base + k;
            const uint32_t stage = fill % kStages;
            const unsigned int tile = __shfl_sync(kFull, claim[k], 0);
            if (lane == 0 && tile < p.n_tiles) claim[k] = atomicAdd(p.work_ctr, 1u);
            if (fill >= (uint32_t)kStages) mbar_wait(bar_empty + 8u * stage, ((fill / kStages) - 1u) & 1u);
            if (tile >= p.n_tiles) {
                /* out of work: sentinel fills end the consumers -- a consumer leaves at the first sentinel slice it is
                   handed, so as many fills as it takes to hand every warp one (they are never released: <= kStages) */
                constexpr uint32_t kSentinels = (NCONS + kTileSlices - 1) / kTileSlices;
                static_assert(kSentinels <= (uint32_t)kStages, "sentinel fills must not wrap the ring");
                for (uint32_t k2 = 0; k2 < kSentinels; k2++) {
                    const uint32_t f2 = fill + k2, st2 = f2 % kStages;
                    if (k2 > 0 && f2 >= (uint32_t)kStages) mbar_wait(bar_empty + 8u * st2, ((f2 / kStages) - 1u) & 1u);
                    if (lane == 0) { s_tile[st2] = kNoTile; mbar_arrive(bar_full + 8u * st2); }
                }
                more = false;
                break;
            }
            const long long off = (long long)tile * kTileBytes;
            const long long avail = exist - off;                     /* > 0 */
            const uint32_t want = kTileBytes + kLook;
            const uint32_t bulk = avail >= (long long)want ? want : (uint32_t)(avail & ~15LL);
            uint8_t *dst = smem_raw + lay.stages + (size_t)stage * kStageBytes;
            if (avail < (long long)want) {
                /* last tile of the buffer: the bytes past the last whole 16 are copied by hand, and the rest of the
                   slice they end in (plus look-ahead) is zero filled so that no lane reads stale shared memory */
                const uint32_t a = (uint32_t)avail;
                uint32_t zend = ((a + (uint32_t)kSliceBytes - 1u) & ~((uint32_t)kSliceBytes - 1u)) + kLook;
                if (zend > want) zend = want;
                for (uint32_t i = bulk + lane; i < zend; i += 32) dst[i] = i < a ? seg[off + i] : (uint8_t)0;
                __syncwarp();
            }
            if (lane == 0) {
                s_tile[stage] = tile;
                if (bulk) {
                    mbar_arrive_expect_tx(bar_full + 8u * stage, bulk);
                    bulk_load(sbase + lay.stages + stage * (uint32_t)kStageBytes, seg + off, bulk, bar_full + 8u * stage);
                } else {
                    mbar_arrive(bar_full + 8u * stage);
                }
            }
        }
    }
    {   /* every claim still in flight must have landed before this CTA reports itself done (the last CTA re-arms the counter) */
        unsigned int sink = 0;
#pragma unroll
        for (int k = 0; k < kClaimDepth; k++) sink |= claim[k];
        if (sink == 0x7fffffffu) s_tile[0] = sink;
    }
}

/* acb_stream_kernel: persistent, one CTA per SM, warp specialised:
 *   producer  (1 warp)          claims tiles from a global counter and keeps the shared-memory ring full
 *                               (cp.async.bulk + mbarrier)
 *   consumers (kConsumers)      take 1 KiB slices from a shared-memory counter: the lane's 32 bytes go to registers, every
 *                               probe position is tested against the gram bitmap in shared memory; the pending bits of all
 *                               lanes become work items spread evenly over the warp, every item reads its text back from
 *                               the stage (still held), probes the tag bitmap (dense key sets) and appends {position,
 *                               anchor tag} to the warp's own candidate list in global memory (the cursor is a register:
 *                               no atomic, a plain store nobody waits for; a list holds a slice's worst case, it cannot
 *                               overflow).  The stage is released, and a warp that has 32 candidates takes them through
 *                               the anchor table (resolve_backlog) while the other warps stream on. */
template <int NW, int STRIDE, int MODE>
__global__ void __launch_bounds__(kFThreads, 1) acb_stream_kernel(const __grid_constant__ ScanParams p) {
    extern __shared__ __align__(128) uint8_t smem_raw[];
    const StreamSmem lay = stream_smem(p.log1);
    const uint32_t sbase = (uint32_t)__cvta_generic_to_shared(smem_raw);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t bar_full = sbase + lay.bars, bar_empty = bar_full + 8u * kStages;
    volatile uint32_t *s_tile = reinterpret_cast<volatile uint32_t *>(smem_raw + lay.tiles);

    {   /* the bitmap -> shared memory with cp.async, so that all of a thread's 16-byte pieces are in flight at once */
        const int n16 = 1 << (p.log1 - 7);
        const uint4 *src = reinterpret_cast<const uint4 *>(p.bm1);
        for (int i = tid; i < n16; i += kFThreads)
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"(sbase + lay.bitmap + 16u * i), "l"(src + i));
        asm volatile("cp.async.commit_group;");
        if (tid < kConsumers) reinterpret_cast<int *>(smem_raw + lay.stage_cnt)[tid] = 0;
        if (tid == 0) *reinterpret_cast<unsigned int *>(smem_raw + lay.next) = 0u;
        if (tid == 0) {
            for (int s = 0; s < kStages; s++) {
                mbar_init(bar_full + 8u * s, 1);                 /* the producer's arrive(.expect_tx) */
                mbar_init(bar_empty + 8u * s, kTileSlices);      /* one arrive per slice */
            }
            asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        }
        asm volatile("cp.async.wait_group 0;" ::: "memory");
    }
    __syncthreads();

    const uint32_t seg_len = (uint32_t)(p.seg_end - p.seg_begin);        /* <= 2^31 */

    if (warp == kConsumers) {
        stream_producer<kConsumers, kTileSlices, kStages>(p, smem_raw, sbase, lay.stages, bar_full, bar_empty, s_tile, lane);
    } else {
        /* ---------------- consumer warps: slice `warp` of every fill */
        ProbeCtx c;
        c.sbm = sbase + lay.bitmap;
        c.n_words = 1u << (p.log1 - 5);
        c.four = 4u + (uint32_t)(p.log1 >> 8);                           /* always 4 */
        c.two = 2u + (uint32_t)(p.log1 >> 8);                            /* always 2 */
        c.sh_bit = 32 - p.log1;
        const uint32_t lt_mask = (1u << lane) - 1u;
        uint32_t mul[NW];
#pragma unroll
        for (int k = 0; k < NW; k++) mul[k] = p.mul1[k];
        uint2 *list = p.cand + ((size_t)blockIdx.x * kConsumers + warp) * kWarpCand;
        uint32_t mul2[NW];
#pragma unroll
        for (int k = 0; k < NW; k++) mul2[k] = p.mul2[k];
        /* the match staging area is idle while the warp streams: it holds the slice's work items (lane << 5 | bit) */
        volatile uint16_t *items = reinterpret_cast<volatile uint16_t *>(smem_raw + lay.stage_rec + (size_t)warp * kStageCap * sizeof(acb_match));
        constexpr int kItemCap = kStageCap * (int)sizeof(acb_match) / 2;
        constexpr int kPendBits = kLaneBytes / STRIDE;
        unsigned int *s_next = reinterpret_cast<unsigned int *>(smem_raw + lay.next);
        unsigned int n_cand = 0;                                         /* warp-uniform */

        /* Slices are handed out dynamically: slice g is slice g % kTileSlices of fill g / kTileSlices.  A warp that is busy
           resolving candidates simply takes fewer slices.  One slice held per warp and slices handed out in order: a
           waiter can never be a whole ring turn ahead of the barrier phase it waits for (kTileSlices above). */
        for (;;) {
            unsigned int g = 0;
            if (lane == 0) g = atomicAdd(s_next, 1u);
            g = __shfl_sync(kFull, g, 0);
            const uint32_t fill = g / (uint32_t)kTileSlices, slice_off = (g % (uint32_t)kTileSlices) * (uint32_t)kSliceBytes;
            const uint32_t stage = fill % (uint32_t)kStages;
            mbar_wait(bar_full + 8u * stage, (fill / (uint32_t)kStages) & 1u);
            const uint32_t tile = s_tile[stage];
            if (tile == kNoTile) break;
            const uint32_t tile_off = tile * (uint32_t)kTileBytes;       /* relative to the segment */
            const uint32_t n_valid = (seg_len - tile_off < (uint32_t)kTileBytes) ? seg_len - tile_off : (uint32_t)kTileBytes;
            if (slice_off < n_valid) {                                   /* warp-uniform */
                const uint32_t slice_saddr = sbase + lay.stages + stage * (uint32_t)kStageBytes + slice_off;
                const uint32_t saddr = slice_saddr + (uint32_t)lane * kLaneBytes;
                uint32_t W[kLaneWords + NW];
#pragma unroll
                for (int i = 0; i < kLaneWords; i += 4) {
                    const uint4 v = lds128(saddr + 4u * i);
                    W[i] = v.x; W[i + 1] = v.y; W[i + 2] = v.z; W[i + 3] = v.w;
                }
                /* look-ahead words: the next lane's first words; lane 31 reads past its slice (next slice / tile pad) */
#pragma unroll
                for (int k = 0; k < NW; k++) W[kLaneWords + k] = __shfl_down_sync(kFull, W[k], 1);
                if (lane == 31) {
#pragma unroll
                    for (int k = 0; k < NW; k++) W[kLaneWords + k] = lds32(saddr + kLaneBytes + 4u * k);
                }
                /* pend: what has to be looked at more closely -- SINGLE: bit i = probe i passed the bitmap;
                   PAIR: bit j = the pair of positions 2j, 2j+1 passed level 1 */
                uint32_t pend;
#ifdef ACB_EXP_NOPROBE
                pend = (W[0] ^ W[3] ^ W[kLaneWords]) == 0x12345678u ? 1u : 0u;      /* timing experiment: the stream skeleton alone */
#else
                pend = probe_single<NW, STRIDE, MODE == kModeWide>(c, W, mul);
#endif
                if (n_valid - slice_off < (uint32_t)kSliceBytes) {       /* last slice of the segment: probes that start past it */
                    const int v = (int)(n_valid - slice_off) - lane * kLaneBytes;
                    const int valid = (v + STRIDE - 1) / STRIDE;
                    pend = (valid <= 0) ? 0u : ((valid >= 32) ? pend : (pend & ((1u << valid) - 1u)));
                }
#ifdef ACB_EXP_NOSURV
                if (pend == 0x9e3779b9u) s_tile[0] = 1u;                 /* timing experiment: probes only, survivors dropped */
                pend = 0;
#endif
                /* The pending bits of all lanes become work items, spread evenly over the warp (a lane's own bits would
                   be worked off one per round: the busiest lane sets the pace); every item reads its text back from the
                   stage, still ours.  A part = the bits whose items fit the staging area at once. */
                if (__ballot_sync(kFull, pend != 0)) {
                    const unsigned int total = __reduce_add_sync(kFull, (unsigned int)__popc(pend));
                    const int nparts = (total > (unsigned int)kItemCap && kPendBits > 8) ? kPendBits / 8 : 1;
                    for (int part = 0; part < nparts; part++) {
                        uint32_t m = nparts > 1 ? ((pend >> (8 * part)) & 0xffu) : pend;
                        const int cnt = __popc(m);
                        int incl = cnt;
#pragma unroll
                        for (int d = 1; d < 32; d <<= 1) {
                            const int v = __shfl_up_sync(kFull, incl, d);
                            if (lane >= d) incl += v;
                        }
                        const int tot = __shfl_sync(kFull, incl, 31);
                        int at = incl - cnt;
                        while (m) {
                            const int bit = __ffs(m) - 1;
                            m &= m - 1;
                            items[at++] = (uint16_t)((lane << 5) | (bit + (nparts > 1 ? 8 * part : 0)));
                        }
                        __syncwarp();
                        for (int base = 0; base < tot; base += 32) {
                            bool ok0 = false;
                            uint32_t pos0 = 0, tag0 = 0;
                            if (base + lane < tot) {
                                const uint32_t it = items[base + lane];
                                const uint32_t t = (it >> 5) * (uint32_t)kLaneBytes + (it & 31u) * (uint32_t)STRIDE;
                                const uint32_t ga = slice_saddr + t, wa = ga & ~3u, sh = (ga & 3u) * 8u;
                                pos0 = tile_off + slice_off + t;
                                {
                                    uint32_t w0 = lds32(wa);
#pragma unroll
                                    for (int k = 0; k < NW; k++) {
                                        const uint32_t w1 = lds32(wa + 4u * (k + 1));
                                        tag0 += __funnelshift_r(w0, w1, sh) * mul2[k];
                                        w0 = w1;
                                    }
                                    tag0 |= 1u;
                                    ok0 = true;
                                }
                            }
                            if (p.log3) {                                  /* large key sets: the tag bitmap in L2 first */
                                const uint32_t i0 = (tag0 * ACB_TAGMAP_MIX) >> (32 - p.log3);
                                if (ok0) ok0 = ((__ldg(p.bm3 + (i0 >> 5)) >> (i0 & 31u)) & 1u) != 0u;
                            }
#ifndef ACB_EXP_NODRAIN
                            /* append {position, hash2 of the gram = the anchor tag} to the warp's candidate list in global
                               memory: the cursor is a register (no atomic), the store is one nobody waits for */
                            const unsigned m0 = __ballot_sync(kFull, ok0);
                            if (ok0) list[n_cand + __popc(m0 & lt_mask)] = make_uint2(pos0, tag0);
                            n_cand += __popc(m0);
#else
                            if (ok0 && tag0 == pos0) s_tile[0] = 2u;      /* timing experiment: candidates dropped */
#endif
                        }
                        __syncwarp();
                    }
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(bar_empty + 8u * stage);          /* this warp is done with the stage */
            /* a full turn of candidates (one per lane): through the anchor table now, while the other warps stream on */
            if (n_cand >= 32u) { resolve_backlog(p, smem_raw, n_cand); n_cand = 0; }
        }
        if (n_cand) resolve_backlog(p, smem_raw, n_cand);
    }
    /* the last CTA to leave re-arms the work counter, so a launch needs no memset before it */
    __syncthreads();
    if (tid == 0) {
        __threadfence();
        unsigned int done = atomicAdd(p.work_ctr + 1, 1u);
        if (done == gridDim.x - 1) {
            p.work_ctr[0] = 0u;
            p.work_ctr[1] = 0u;
            __threadfence();
        }
    }
}

/* ------------------------------------------------------------ the pair kernel
 * acb_pair_kernel: the stream kernel of the PAIR placement (gram 4, stride 1, 1-byte letters; acb_hash.h).  Same
 * producer, same dynamic slices, a ring of its own (kPairTileSlices x kPairStages); what differs is everything a
 * consumer warp does with its slice:
 *   level 1   one shared-memory word per PAIR of positions, selected by the three bytes the pair's grams share; the
 *             word holds one bit per (role, remaining byte), so the loop leaves a per-POSITION pass mask -- 9.5
 *             instructions per pair, 2 % of the positions pass on random text against 10 k keys.  A lane owns two runs
 *             of 16 bytes (16 * lane and 512 + 16 * lane of the slice): both 16-byte loads of a warp are conflict free;
 *   items     while the stage is held: the pending positions of all lanes are pushed into a list in shared memory
 *             (ballot rounds) and worked off 32 at a time -- the gram read back from the stage, the anchor tag
 *             (hash 2), level 2 (shared memory, two bits keyed by the tag); survivors ({position, tag}) go to the
 *             warp's candidate ring in SHARED memory (no global list, no round trip).  A round never takes more items
 *             than the ring has room for, so the stage is not held across an anchor look-up unless one slice alone
 *             overflows the ring;
 *   resolve   after the release, as soon as the ring holds 32 entries -- one per lane: the text at the position and
 *             the anchor slot of the tag are loaded together (L2), UNIQUE keys are compared in registers, the hits of
 *             the warp take ONE atomicAdd on the record counter and are stored straight to the record buffer (no
 *             staging copy); MULTI anchors (keys sharing their first four bytes) take the general path with one
 *             atomic per record. */
#ifndef ACB_PAIR_CONSUMERS
#define ACB_PAIR_CONSUMERS 27
#endif
constexpr int kPairConsumers = ACB_PAIR_CONSUMERS;          /* consumer warps of the pair kernel: 27 + the producer = 896 threads leave 72 registers per thread,
                                                                and the level-1 loop stops spilling (31 consumers at 64 registers: 4 % slower on C2) */
constexpr int kPairThreads = (kPairConsumers + 1) * 32;
/* The pair kernel's ring: power-of-two tiles and stages, so that a slice number splits into fill, slice, stage and
 * barrier phase by shifts and masks.  32 KiB tiles x 2 stages: the 27 consumer warps work inside one tile while the
 * next one loads.  Fastest of the shapes that fit next to the 144 KiB filter on the H100 (DESIGN 4.1 has the sweep). */
#ifndef ACB_PAIR_TILE_SLICES
#define ACB_PAIR_TILE_SLICES 32
#endif
#ifndef ACB_PAIR_STAGES
#define ACB_PAIR_STAGES 2
#endif
constexpr int kPairTileSlices = ACB_PAIR_TILE_SLICES;
constexpr int kPairStages     = ACB_PAIR_STAGES;
constexpr int kPairTileLog    = __builtin_ctz(kPairTileSlices);
constexpr int kPairStageLog   = __builtin_ctz(kPairStages);
constexpr int kPairTileBytes  = kPairTileSlices * kSliceBytes;
constexpr int kPairStageBytes = (kPairTileBytes + kLook + 127) / 128 * 128;
static_assert((kPairTileSlices & (kPairTileSlices - 1)) == 0 && (kPairStages & (kPairStages - 1)) == 0 && kSliceBytes == 1024,
              "pair ring: power-of-two tiles and stages of 1 KiB slices");
static_assert((kPairConsumers + kPairTileSlices - 1) / kPairTileSlices + 2 < 2 * kPairStages && kPairThreads <= 1024, "pair kernel shape");
constexpr int kPairRing = 64;                                /* candidate ring entries per consumer warp */
constexpr int kPairItems = 64;                               /* item list entries (uint16 byte offsets in the slice) per consumer warp */
static_assert(kPairRing >= 31 + 32, "a one-round slice must fit the ring next to a turn not yet resolved");

/* The fields of ScanParams a resolve turn reads, copied to shared memory once per CTA.  pair_resolve is not inlined,
 * so it would see the parameter block only through a generic pointer: every field a generic load (LD.E), several of
 * them one after another on the turn's critical path.  From shared memory they are LDS.128 of 16-byte groups, in the
 * order the turn needs them: the text and the anchor slot, attributing a hit, storing the records. */
struct PairTurnArgs {
    const uint8_t *hay;                                   /* group 0 */
    long long total;
    long long seg_begin;                                  /* group 1 */
    const uint4 *anchors;
    int logA, stride_shift, letter_shift, pad;            /* group 2 */
    const long long *offsets;                             /* group 3 */
    long long n_hay;
    long long stride_bytes;                               /* group 4 */
    long long cap;
    acb_match *out;                                       /* group 5 */
    unsigned long long *count;
};
static_assert(sizeof(PairTurnArgs) == 96, "PairTurnArgs is six 16-byte groups");

struct PairSmem {
    uint32_t bitmap, bitmap2, stages, ring, items, args, bars, tiles, next, total;
};
__host__ __device__ inline PairSmem pair_smem(int log1, int log2b) {
    PairSmem s;
    uint32_t o = 0;
    s.bitmap = o;    o += 1u << (log1 - 3);                       /* >= 1 KiB: level 2 follows without a gap, as in bm1 */
    s.bitmap2 = o;   o += 1u << (log2b - 3);                      o = (o + 127u) & ~127u;
    s.stages = o;    o += (uint32_t)kPairStages * kPairStageBytes;
    s.ring = o;      o += (uint32_t)kPairConsumers * kPairRing * 8u;
    s.items = o;     o += (uint32_t)kPairConsumers * kPairItems * 2u;
    s.bars = o;      o += 2u * kPairStages * 8u;
    s.tiles = o;     o += (uint32_t)kPairStages * 4u;
    s.next = o;      o += 4u;                                     o = (o + 15u) & ~15u;
    /* last, so that pair_resolve finds it from the launch's dynamic shared memory size, without an argument (at offset
       0 it moved the bitmap and the stages by 128 bytes, which cost the streaming skeleton 1.6 us per C2 launch) */
    s.args = o;      o += (uint32_t)sizeof(PairTurnArgs);
    s.total = o;
    return s;
}

__device__ __forceinline__ void emit_direct(const ScanParams &p, int32_t h, int32_t e, int32_t k) {
    const unsigned long long g = atomicAdd(p.count, 1ULL);
    if (g < (unsigned long long)p.cap) { acb_match m; m.hay_id = h; m.end_index = e; m.key_id = k; p.out[g] = m; }
}

/* the general way through the anchor table from `slot` on (resolve_chain's loop), records emitted one by one */
__device__ __noinline__ void pair_resolve_general(const ScanParams &p, long long q, uint32_t tag, uint32_t slot, uint4 e0, uint4 e1) {
    const uint32_t amask = (1u << p.logA) - 1u;
    long long h = -1, hs = 0, he = 0;
    for (;;) {
        if (e0.x == 0u) break;
        if (e0.x == tag) {
            const uint32_t kw[5] = {e0.w, e1.x, e1.y, e1.z, e1.w};
            const int j = (int)(e0.z & 0xffu), len = (int)((e0.z >> 8) & 0xffu);
            const int32_t kid = (int32_t)e0.y;
            if (h < 0) find_haystack(p, q, h, hs, he);
            const long long start = q - j;
            if (start >= hs && start + len <= he) {
                uint32_t ts[6];
                load_text(p, start, ts);
                if (text_equals(ts, start, len, kw)) {
                    if (kid >= 0) {
                        emit_direct(p, (int32_t)h, (int32_t)(((start + len - hs) >> p.letter_shift) - 1), kid);
                    } else {                                           /* MULTI: exact gram, then the trie from the root */
                        int32_t st = 0;
                        for (long long i = start; i < he; ++i) {
                            const int c = __ldg(p.cls + p.hay[i]);
                            const int32_t nx = __ldg(p.gto + (long long)c * p.S + st);
                            if (nx < 0) break;
                            st = nx & kIdMask;
                            if (nx & kTermBit) emit_direct(p, (int32_t)h, (int32_t)((i - hs + 1) / p.L - 1), __ldg(p.key_of + st));
                        }
                    }
                }
            }
            if (e0.z & 0x10000u) break;
        }
        slot = (slot + 1) & amask;
        e0 = __ldg(p.anchors + 2 * (size_t)slot);
        e1 = __ldg(p.anchors + 2 * (size_t)slot + 1);
    }
}

/* groups [g0, g1) of the pair kernel's PairTurnArgs (the last bytes of its shared memory), loaded where the turn needs
 * them: all of them at once would hold 24 registers through the turn, more than the streaming loop leaves a callee.
 * The block is written once, before the kernel's first __syncthreads. */
union PairTurnRegs {
    uint4 v[sizeof(PairTurnArgs) / 16];
    PairTurnArgs a;
};
__device__ __forceinline__ void load_turn_args(PairTurnRegs &u, int g0, int g1) {
    extern __shared__ __align__(128) uint8_t smem_raw[];
    uint32_t dyn;
    asm("mov.u32 %0, %%dynamic_smem_size;" : "=r"(dyn));
    const uint32_t saddr = (uint32_t)__cvta_generic_to_shared(smem_raw) + dyn - (uint32_t)sizeof(PairTurnArgs);
#pragma unroll
    for (int i = g0; i < g1; i++)
        asm("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(u.v[i].x), "=r"(u.v[i].y), "=r"(u.v[i].z), "=r"(u.v[i].w) : "r"(saddr + 16u * i));
}

/* one turn of a warp's candidates (ring entries head .. head + n - 1, n <= 32, one per lane) through the anchor table.
 * Not inlined: the streaming loop keeps its registers and its schedule, and this runs once per five slices or so.
 * Its fields come from the PairTurnArgs in shared memory; `p` is only handed on to the general path. */
__device__ __noinline__ void pair_resolve(const ScanParams &p, uint32_t sring, unsigned int head, unsigned int n) {
    const int lane = threadIdx.x & 31;
    const uint32_t lt_mask = (1u << lane) - 1u;
    PairTurnRegs u;
    const PairTurnArgs &a = u.a;
    bool hit = false;
    int32_t rh = 0, re = 0, rk = 0;
    if ((unsigned)lane < n) {
        load_turn_args(u, 0, 3);
        const uint32_t amask = (1u << a.logA) - 1u;
        const uint2 e = lds64(sring + (((head + (unsigned)lane) & (kPairRing - 1u)) << 3));
        const long long q = a.seg_begin + (long long)e.x;
        /* one round trip for both: the anchor slot and the text are issued before either is used */
        uint32_t slot = e.y >> (32 - a.logA);
        uint4 e0 = __ldg(a.anchors + 2 * (size_t)slot), e1 = __ldg(a.anchors + 2 * (size_t)slot + 1);
        uint32_t tq[6];
        load_text(a, q, tq);
        while (e0.x != 0u && e0.x != e.y) {                      /* a foreign tag in the way: linear probing */
            slot = (slot + 1) & amask;
            e0 = __ldg(a.anchors + 2 * (size_t)slot);
            e1 = __ldg(a.anchors + 2 * (size_t)slot + 1);
        }
        if (e0.x != 0u) {
            if ((int32_t)e0.y >= 0 && (e0.z & 0x100ffu) == 0x10000u) {   /* the tag's ONE entry: UNIQUE, anchored at its first byte */
                const uint32_t kw[5] = {e0.w, e1.x, e1.y, e1.z, e1.w};
                const int len = (int)((e0.z >> 8) & 0xffu);
                long long h, hs, he;
                load_turn_args(u, 3, 5);
                find_haystack(a, q, h, hs, he);
                hit = q + len <= he && text_equals(tq, q, len, kw);
                rh = (int32_t)h;
                re = (int32_t)(((q + len - hs) >> a.letter_shift) - 1);
                rk = (int32_t)e0.y;
            } else {
                pair_resolve_general(p, q, e.y, slot, e0, e1);
            }
        }
    }
    /* the hits of the warp: ONE atomic on the record counter, records stored straight to the record buffer (both
       global-space operations: a.count and a.out are generic pointers to the compiler) */
    load_turn_args(u, 4, 6);
    const unsigned mh = __ballot_sync(kFull, hit);
    if (mh) {
        unsigned long long base = 0;
        if (lane == 0)
            asm volatile("atom.global.add.u64 %0, [%1], %2;" : "=l"(base) : "l"(__cvta_generic_to_global(a.count)), "l"((unsigned long long)__popc(mh)) : "memory");
        base = __shfl_sync(kFull, base, 0) + (unsigned long long)__popc(mh & lt_mask);
        if (hit && base < (unsigned long long)a.cap)
            asm volatile("st.global.u32 [%0], %1;\n\tst.global.u32 [%0+4], %2;\n\tst.global.u32 [%0+8], %3;"   /* 12-byte records: 4-byte aligned */
                         :: "l"(__cvta_generic_to_global(a.out + base)), "r"(rh), "r"(re), "r"(rk) : "memory");
    }
}

/* level 1 of one 16-byte run (words R[0..3], look-ahead word R[4]): the pass bits of its 16 positions are shifted
 * into acc, first position first (acb_hash.h, PAIR placement).  Per pair: the window at x+1, ONE 64-bit multiply (low
 * half -> word index, high half -> role 1's bit), the word, and per role a left shift that brings the tested bit to
 * bit 31 plus a one-bit funnel shift that moves it into the mask. */
__device__ __forceinline__ uint32_t probe_pair_run(uint32_t acc, uint32_t sbm, uint32_t n_words, uint32_t four, const uint32_t (&R)[5], uint32_t mulp) {
#pragma unroll
    for (int x = 0; x < 16; x += 2) {
#ifdef ACB_EXP_L1_NOWIDE
        const uint32_t hc = window(R, x + 1) * mulp, hb = hc >> 7;
#else
        const unsigned long long pr = mul_wide(window(R, x + 1), mulp);
        const uint32_t hc = (uint32_t)pr, hb = (uint32_t)(pr >> 32);
#endif
#ifdef ACB_EXP_L1_SHIFTIDX
        const uint32_t waddr = (hc >> 17) * four + sbm;
#else
        const uint32_t waddr = __umulhi(hc, n_words) * four + sbm;
#endif
#ifdef ACB_EXP_L1_NOLDS
        const uint32_t word = waddr;
#else
        const uint32_t word = lds_bitmap(waddr);
#endif
        const uint32_t ta = __funnelshift_l(0u, word, window(R, x));      /* word << (text[x] & 31): role 0's bit -> bit 31 */
        const uint32_t tb = __funnelshift_l(0u, word, hb);                /* role 1's */
#ifdef ACB_L1_CARRY
        asm("{ .reg .u32 t2; add.cc.u32 t2, %1, %1; addc.u32 %0, %0, %0; add.cc.u32 t2, %2, %2; addc.u32 %0, %0, %0; }"
            : "+r"(acc) : "r"(ta), "r"(tb));
#else
        acc = __funnelshift_l(ta, acc, 1);                                /* acc << 1 | bit 31 of ta */
        acc = __funnelshift_l(tb, acc, 1);
#endif
    }
    return acc;
}

template <int L2B>
__global__ void __launch_bounds__(kPairThreads, 1) acb_pair_kernel(const __grid_constant__ ScanParams p) {
    extern __shared__ __align__(128) uint8_t smem_raw[];
    const PairSmem lay = pair_smem(p.log1, p.log2b);
    const uint32_t sbase = (uint32_t)__cvta_generic_to_shared(smem_raw);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t bar_full = sbase + lay.bars, bar_empty = bar_full + 8u * kPairStages;
    volatile uint32_t *s_tile = reinterpret_cast<volatile uint32_t *>(smem_raw + lay.tiles);

    if (tid == 0) {
        *reinterpret_cast<unsigned int *>(smem_raw + lay.next) = 0u;
        /* the resolve turn's fields (written in the consumers' prologue instead, the copy measured 0.9 us slower per C2 launch) */
        PairTurnArgs &a = *reinterpret_cast<PairTurnArgs *>(smem_raw + lay.args);
        a.hay = p.hay; a.total = p.total; a.seg_begin = p.seg_begin; a.anchors = p.anchors;
        a.logA = p.logA; a.stride_shift = p.stride_shift; a.letter_shift = p.letter_shift; a.pad = 0;
        a.offsets = p.offsets; a.n_hay = p.n_hay; a.stride_bytes = p.stride_bytes; a.cap = p.cap;
        a.out = p.out; a.count = p.count;
        for (int s = 0; s < kPairStages; s++) {
            mbar_init(bar_full + 8u * s, 1);
            mbar_init(bar_empty + 8u * s, kPairTileSlices);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    const uint32_t seg_len = (uint32_t)(p.seg_end - p.seg_begin);        /* <= 2^31 */

    if (warp == kPairConsumers) {
        /* the producer starts at once: the first tiles are on their way while the consumers fetch the bitmap */
        stream_producer<kPairConsumers, kPairTileSlices, kPairStages>(p, smem_raw, sbase, lay.stages, bar_full, bar_empty, s_tile, lane);
    } else {
        {   /* both levels of the bitmap -> shared memory with cp.async, by the consumer warps (named barrier 1) */
            const int n16 = (1 << (p.log1 - 7)) + (1 << (p.log2b - 7));
            const uint4 *src = reinterpret_cast<const uint4 *>(p.bm1);
            for (int i = tid; i < n16; i += kPairConsumers * 32)
                asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"(sbase + lay.bitmap + 16u * i), "l"(src + i));
            asm volatile("cp.async.commit_group;");
            asm volatile("cp.async.wait_group 0;" ::: "memory");
            asm volatile("bar.sync 1, %0;" :: "n"(kPairConsumers * 32) : "memory");
        }
        const uint32_t sbm = sbase + lay.bitmap, sbm2 = sbase + lay.bitmap2;
        const uint32_t n_words = 1u << (p.log1 - 5);                     /* umulhi(hc, n_words) = hc >> (37 - log1) on the FMA pipe */
        const int l2b = L2B ? L2B : p.log2b;                             /* L2B != 0: compile-time shifts */
        const int shy_w = 37 - l2b, shy_a = 32 - l2b, shy_b = 27 - l2b;
        const uint32_t four = 4u + (uint32_t)(p.log1 >> 8);              /* always 4, opaque: the address is one IMAD */
        const uint32_t mulp = acb_pair_mul() + (uint32_t)(p.log1 >> 8);
        const uint32_t mul2 = p.mul2[0];
        const uint32_t lt_mask = (1u << lane) - 1u;
        const uint32_t sring = sbase + lay.ring + (uint32_t)warp * (kPairRing * 8u);
        const uint32_t sitems = sbase + lay.items + (uint32_t)warp * (kPairItems * 2u);
        const uint32_t snext = sbase + lay.next;
        const uint32_t sstages = sbase + lay.stages;
        const uint32_t lane16 = (uint32_t)lane << 4;
        unsigned int n_cand = 0, head = 0;                               /* warp-uniform: entries [head, head + n_cand) of the ring */

        /* bit y of a lane's pending mask is position y of its first 16-byte run, or y - 16 of its second: byte
           16 * lane + y (+ 496) of the slice */
        auto offset_of = [&](uint32_t y) { return lane16 + y + (y & 16u) * 31u; };
        auto top_bit = [](uint32_t m) { uint32_t y; asm("bfind.u32 %0, %1;" : "=r"(y) : "r"(m)); return y; };   /* m != 0 */
        /* the list: every lane writes the byte offsets of its pending positions after those of the lanes below it */
        auto list_all = [&](uint32_t pend) {
            const unsigned int cnt = (unsigned)__popc(pend);
            unsigned int incl = cnt;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const unsigned int v = __shfl_up_sync(kFull, incl, d);
                if (lane >= d) incl += v;
            }
            uint32_t at = sitems + 2u * (incl - cnt);
            while (pend) {
                const uint32_t y = top_bit(pend);
                pend ^= 1u << y;
                sts16(at, offset_of(y));
                at += 2u;
            }
        };
        /* one round of items, list entries [base, base + take) with take <= 32, one per lane: the gram read back from
           the stage, the anchor tag (hash 2), level 2; the survivors {position, tag} go to the candidate ring, which
           has room for `take` more */
        auto item_round = [&](uint32_t slice_saddr, uint32_t pos_base, unsigned int base, unsigned int take) {
            uint32_t ok = 0, pos = 0, tag = 0;
            if ((unsigned)lane < take) {
                const uint32_t t = lds16(sitems + 2u * (base + (unsigned)lane));
                const uint32_t ga = slice_saddr + t, wa = ga & ~3u;
                const uint32_t lo = lds32(wa), hi = lds32(wa + 4u);
                const uint32_t w = __funnelshift_r(lo, hi, ga << 3);                    /* wrap shift: (ga & 3) * 8 */
                tag = (w * mul2) | 1u;
                const uint32_t word = lds_bitmap((tag >> shy_w) * four + sbm2);
                ok = __funnelshift_r(word, 0u, tag >> shy_a) & __funnelshift_r(word, 0u, tag >> shy_b) & 1u;
                pos = pos_base + t;
            }
            if (p.log3) {                                                /* very large key sets: the tag bitmap in L2 as well */
                const uint32_t i0 = (tag * ACB_TAGMAP_MIX) >> (32 - p.log3);
                if (ok) ok = (__ldg(p.bm3 + (i0 >> 5)) >> (i0 & 31u)) & 1u;
            }
#ifdef ACB_EXP_NODRAIN
            if (ok && tag == pos) s_tile[0] = 2u;
#else
            const unsigned mk = __ballot_sync(kFull, ok);
            if (ok) {
                const uint32_t at = sring + (((head + n_cand + (unsigned)__popc(mk & lt_mask)) & (kPairRing - 1u)) << 3);
                asm volatile("st.shared.v2.u32 [%0], {%1, %2};" :: "r"(at), "r"(pos), "r"(tag) : "memory");
            }
            n_cand += (unsigned)__popc(mk);
#endif
        };

        for (;;) {
            /* slice g is slice g % kPairTileSlices of fill g / kPairTileSlices.  One lane claims it; elect.sync tells
               ptxas that one lane does, so the atomic is not wrapped in warp aggregation */
            unsigned int g = 0;
            asm volatile("{ .reg .pred e; elect.sync _|e, 0xffffffff; @e atom.shared.add.u32 %0, [%1], 1; }"
                         : "+r"(g) : "r"(snext) : "memory");
            g = __shfl_sync(kFull, g, 0);
            const uint32_t fill = g >> kPairTileLog, stage = fill & (kPairStages - 1u);
            const uint32_t slice_off = (g & (kPairTileSlices - 1u)) * (uint32_t)kSliceBytes;
            mbar_wait(bar_full + 8u * stage, (fill >> kPairStageLog) & 1u);
            const uint32_t tile = s_tile[stage];
            if (tile == kNoTile) break;
            const uint32_t tile_off = tile * (uint32_t)kPairTileBytes;   /* relative to the segment */
            const uint32_t n_valid = (seg_len - tile_off < (uint32_t)kPairTileBytes) ? seg_len - tile_off : (uint32_t)kPairTileBytes;
            const uint32_t slice_saddr = sstages + stage * (uint32_t)kPairStageBytes + slice_off;
            const uint32_t pos_base = tile_off + slice_off;
            uint32_t pend = 0;       /* bit y < 16: position 16 * lane + y of the slice passed level 1; y >= 16: position 512 + 16 * lane + y - 16 */
            if (slice_off < n_valid) {                                   /* warp-uniform */
                const uint32_t saddr = slice_saddr + lane16;
                uint32_t R0[5], R1[5];
                {
                    const uint4 v = lds128(saddr), u = lds128(saddr + 512u);
                    R0[0] = v.x; R0[1] = v.y; R0[2] = v.z; R0[3] = v.w;
                    R1[0] = u.x; R1[1] = u.y; R1[2] = u.z; R1[3] = u.w;
                }
                /* look-ahead words: the next lane's first word of the same run; lane 31's are lane 0's first word of the
                   second run and the first word after the slice (next slice / tile pad) */
                R0[4] = __shfl_down_sync(kFull, R0[0], 1);
                R1[4] = __shfl_down_sync(kFull, R1[0], 1);
                const uint32_t r1_first = __shfl_sync(kFull, R1[0], 0);
                if (lane == 31) { R0[4] = r1_first; R1[4] = lds32(slice_saddr + (uint32_t)kSliceBytes); }
#ifdef ACB_EXP_NOPROBE
                pend = (R0[0] ^ R0[3] ^ R0[4] ^ R1[1] ^ R1[4]) == 0x12345678u ? 1u : 0u;
#else
                pend = probe_pair_run(0u, sbm, n_words, four, R0, mulp);
                pend = probe_pair_run(pend, sbm, n_words, four, R1, mulp);
                pend = __brev(pend);
#endif
                if (n_valid - slice_off < (uint32_t)kSliceBytes) {       /* last slice of the segment: positions past its end */
                    const int v0 = (int)(n_valid - slice_off) - lane * 16, v1 = v0 - 512;
                    const uint32_t m0 = v0 <= 0 ? 0u : (v0 >= 16 ? 0xffffu : ((1u << v0) - 1u));
                    const uint32_t m1 = v1 <= 0 ? 0u : (v1 >= 16 ? 0xffffu : ((1u << v1) - 1u));
                    pend &= m0 | (m1 << 16);
                }
#ifdef ACB_EXP_NOSURV
                if (pend == 0x9e3779b9u) s_tile[0] = 1u;
                pend = 0;
#endif
            }
            /* items: the pending positions of all lanes go to the list and are worked off 32 at a time */
            unsigned int tot = __reduce_add_sync(kFull, (unsigned)__popc(pend));
            if (tot <= 32u) {
                /* the common case, one round: fewer than 32 candidates are waiting (they are resolved after every
                   slice that brings them to 32), so the ring has room for all of them */
                if (tot) {
                    list_all(pend);
                    __syncwarp();
                    item_round(slice_saddr, pos_base, 0u, tot);
                }
            } else {
                /* more than one round (dense text): passes of at most the list's size -- the whole list placed by the
                   scan, or, past kPairItems, ballot rounds of one position per lane -- and rounds that never take more
                   items than the ring has room for */
                while (tot) {
                    unsigned int n_items;
                    if (tot <= (unsigned)kPairItems) {
                        list_all(pend);
                        n_items = tot;
                        tot = 0;
                    } else {
                        n_items = 0;
                        do {
                            const unsigned int mp = __ballot_sync(kFull, pend != 0u);
                            if (pend) {
                                const uint32_t y = top_bit(pend);
                                pend ^= 1u << y;
                                sts16(sitems + 2u * (n_items + (unsigned)__popc(mp & lt_mask)), offset_of(y));
                            }
                            n_items += (unsigned)__popc(mp);
                        } while (n_items <= (unsigned)(kPairItems - 32));
                        tot -= n_items;
                    }
                    __syncwarp();
                    for (unsigned int base = 0; base < n_items;) {
                        if (n_cand == (unsigned)kPairRing) {            /* one slice alone filled the ring */
                            __syncwarp();                                /* the entries were written by other lanes */
                            pair_resolve(p, sring, head, 32u); head += 32u; n_cand -= 32u;
                            continue;
                        }
                        unsigned int take = n_items - base;
                        if (take > 32u) take = 32u;
                        if (take > (unsigned)kPairRing - n_cand) take = (unsigned)kPairRing - n_cand;
                        item_round(slice_saddr, pos_base, base, take);
                        base += take;
                    }
                    __syncwarp();
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(bar_empty + 8u * stage);          /* this warp is done with the stage */
            /* a full turn of candidates (one per lane): through the anchor table now, while the other warps stream on */
            while (n_cand >= 32u) { pair_resolve(p, sring, head, 32u); head += 32u; n_cand -= 32u; }
        }
        if (n_cand) { __syncwarp(); pair_resolve(p, sring, head, n_cand); }
    }
    /* the last CTA to leave re-arms the work counter, so a launch needs no memset before it */
    __syncthreads();
    if (tid == 0) {
        __threadfence();
        unsigned int done = atomicAdd(p.work_ctr + 1, 1u);
        if (done == gridDim.x - 1) {
            p.work_ctr[0] = 0u;
            p.work_ctr[1] = 0u;
            __threadfence();
        }
    }
}

/* ---------------------------------------------------------- the DFA kernel */

__global__ void __launch_bounds__(kDfaThreads) acb_dfa_kernel(const ScanParams p) {
    const long long span = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long a = span * kDfaSpan;
    if (a >= p.total) return;
    const long long b = (a + kDfaSpan < p.total) ? a + kDfaSpan : p.total;
    long long h, hs, he;
    find_haystack(p, a, h, hs, he);
    /* with variable offsets, position a may sit in a run of empty haystacks: find_haystack
       returns the last h with offsets[h] <= a, which is the non-empty one containing a */
    long long i = a - p.max_key_bytes;               /* warm-up start, letter aligned */
    if (i < hs) i = hs;
    int32_t st = 0;
    const int L = p.L;
    for (; i < b; ++i) {
        while (i >= he) {                             /* crossed into the next haystack(s) */
            h += 1; hs = he;
            he = (p.offsets == nullptr) ? hs + p.stride_bytes : __ldg(p.offsets + h + 1);
            st = 0;
        }
        const long long col = (long long)__ldg(p.cls + p.hay[i]) * p.S;
        int32_t nx;
        while ((nx = __ldg(p.gto + col + st)) < 0 && st != 0) st = __ldg(p.fail + st);   /* src/trie.c:182-190 */
        st = (nx < 0) ? 0 : (nx & kIdMask);
        if (i >= a && st != 0 && ((i + 1 - hs) % L) == 0) {
            const int32_t o0 = __ldg(p.out_ptr + st), o1 = __ldg(p.out_ptr + st + 1);
            for (int32_t o = o0; o < o1; ++o) {
                const int32_t k = __ldg(p.out_idx + o);
                const long long kb = (long long)__ldg(p.key_len + k) * L;
                if (i + 1 - kb < hs) continue;        /* cannot happen (state resets at hs); defensive */
                unsigned long long g = atomicAdd(p.count, 1ULL);
                if (g < (unsigned long long)p.cap) {
                    acb_match m;
                    m.hay_id = (int32_t)h;
                    m.end_index = (int32_t)((i - hs + 1) / L - 1);
                    m.key_id = k;
                    p.out[g] = m;
                }
            }
        }
    }
}

/* ------------------------------------------------------- the iter_long kernel */
/* ACB_ALGO_LONG: the reference's longest-match iterator (src/AutomatonSearchIterLong.c:89-153) is a
 * sequential state machine per haystack (after every reported match it restarts from the root at the
 * match's last letter), so one lane replays it per haystack: trie edges only (`goto`, letter by letter),
 * letter-level fail links, and the reference's early return when a non-terminal state's fail state ends
 * a key (:122-126).  Records of one haystack come out in increasing end_index. */
__device__ __forceinline__ int32_t letter_step(const ScanParams &p, int32_t st, const uint8_t *letter) {
    for (int b = 0; b < p.L; b++) {
        const int32_t nx = __ldg(p.gto + (long long)__ldg(p.cls + letter[b]) * p.S + st);
        if (nx < 0) return -1;
        st = nx & kIdMask;
    }
    return st;
}

__global__ void __launch_bounds__(kDfaThreads) acb_long_kernel(const __grid_constant__ ScanParams p) {
    const long long h = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (h >= p.n_hay) return;
    const long long hs = p.offsets ? __ldg(p.offsets + h) : h * p.stride_bytes;
    const long long he = p.offsets ? __ldg(p.offsets + h + 1) : hs + p.stride_bytes;
    const long long n = (he - hs) / p.L;                       /* letters */
    const uint8_t *text = p.hay + hs;
    int32_t state = p.long_start ? __ldg(p.long_start + h) : ((h == 0) ? p.long_init : 0), last_node = -1;   /* the walk of a stream goes on where the last chunk left it */
    long long index = -1, last_index = -1;
    for (;;) {
        if (last_node >= 0) {                                   /* return_output */
            unsigned long long g = atomicAdd(p.count, 1ULL);
            if (g < (unsigned long long)p.cap) {
                acb_match m;
                m.hay_id = (int32_t)h;
                m.end_index = (int32_t)last_index;
                m.key_id = __ldg(p.key_of + last_node);
                p.out[g] = m;
            }
            state = 0;                                          /* start over: no overlapped results */
            index = last_index;
            last_node = -1;
            last_index = -1;
        }
        index += 1;
        bool emit = false;
        while (index < n) {
            const int32_t nx = letter_step(p, state, text + index * p.L);
            if (nx >= 0) {
                if (__ldg(p.key_of + nx) >= 0) {
                    last_node = nx;
                    last_index = index;
                } else {
                    const int32_t fl = __ldg(p.letter_fail + nx);
                    if (fl > 0 && __ldg(p.key_of + fl) >= 0) { last_node = fl; last_index = index; emit = true; break; }
                }
                state = nx;
                index += 1;
            } else {
                if (last_node >= 0) { emit = true; break; }
                for (;;) {
                    state = __ldg(p.letter_fail + state);
                    if (state < 0) { state = 0; index += 1; break; }
                    if (letter_step(p, state, text + index * p.L) >= 0) break;
                }
            }
        }
        if (!emit && last_node < 0) break;                      /* StopIteration */
    }
    if (h == 0 && p.long_final) *p.long_final = state;
    if (p.long_end) p.long_end[h] = state;
}

__global__ void acb_flag_goto_kernel(int32_t *gto, const int32_t *key_of, size_t n) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const int32_t v = gto[i];
        if (v >= 0 && key_of[v] >= 0) gto[i] = v | kTermBit;
    }
}

} // namespace

/* ------------------------------------------------------------- the table */

/* Scratch that the last call's work, on any CUDA stream, may still read (scratch_take, carve, scratch_done) */
struct Scratch {
    void *buf = nullptr; size_t cap = 0;
    cudaEvent_t done = nullptr;              /* the last call's work on buf has been issued before it */
    void release() { cudaFree(buf); if (done) cudaEventDestroy(done); }
};

struct acb_table {
    int device = 0;
    int sm_count = 0;                        /* sizes the per-CTA allocations (d_cand); launches take grid_sms() */
    int32_t S = 0, K = 0, L = 1, n_keys = 0, gram = 1, stride = 1, log1 = 13, log3 = 0, logA = 10, filter_flags = 0, log2b = 0;
    int32_t min_key_bytes = 0, max_key_bytes = 0;
    uint32_t mul1[ACB_MAX_WINDOWS], mul2[ACB_MAX_WINDOWS];
    uint8_t *d_cls = nullptr;
    int32_t *d_lfail = nullptr;
    int32_t *d_goto = nullptr, *d_fail = nullptr, *d_keyof = nullptr, *d_outptr = nullptr, *d_outidx = nullptr, *d_keylen = nullptr;
    uint32_t *d_bm1 = nullptr, *d_bm3 = nullptr, *d_anchors = nullptr;
    unsigned int *d_work = nullptr;
    uint2 *d_cand = nullptr;                 /* candidate lists of the stream kernel's consumer warps (kWarpCand entries each) */
    int32_t long_init = 0;                   /* iter_long streaming: start state of haystack 0 of the next ACB_ALGO_LONG scan */
    int32_t *d_long_final = nullptr;         /* ... and the state it ended in */
    int32_t long_final_host = -1;            /* that state when the last ACB_ALGO_LONG scan launched nothing, else -1 */
    long long dev_bytes = 0;
    std::vector<int32_t> key_len;            /* host copy, for sorting records */
    /* workspace of acb_scan_host */
    cudaStream_t stream = nullptr, s_copy = nullptr, s_sort = nullptr;      /* compute; H2D of the pipelined host scan; sort + D2H */
    std::vector<cudaEvent_t> ev_h2d, ev_scan;                               /* per chunk of the pipelined host scan */
    unsigned long long *h_counts = nullptr; size_t h_counts_cap = 0;        /* pinned: record count after every chunk */
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    uint8_t *w_hay = nullptr; size_t w_hay_cap = 0;
    long long *w_off = nullptr; size_t w_off_cap = 0;
    acb_match *w_out = nullptr; size_t w_out_cap = 0;
    unsigned long long *w_count = nullptr;
    unsigned long long *h_count = nullptr;   /* pinned */
    acb_match *h_out = nullptr; size_t h_out_cap = 0;   /* pinned staging for the records */
    unsigned long long h_out_n = 0;                      /* records of the last scan held in h_out */
    Scratch sort_buf;                                    /* the record sort: keys, sorted records, cub scratch */
    /* workspace of the white-space scans (acb_scan_*_skip, stream batches with a skip set) */
    uint8_t *k_buf = nullptr; size_t k_buf_cap = 0;      /* the compacted letters */
    uint32_t *k_mask = nullptr; size_t k_mask_cap = 0;   /* keep bit per letter, one word per 32-letter group */
    uint16_t *k_gpre = nullptr; size_t k_gpre_cap = 0;   /* kept letters before the group, within its tile */
    long long *k_tile_pre = nullptr; size_t k_tile_pre_cap = 0;   /* kept letters before the tile; [n_tiles] = all */
    unsigned long long *k_status = nullptr; size_t k_status_cap = 0;   /* decoupled look-back */
    long long *k_coff = nullptr; size_t k_coff_cap = 0;  /* compacted byte offsets of the haystacks */
    uint32_t *k_set = nullptr;                           /* the skip set (ACB_MAX_SKIP) */
    unsigned int *k_ctr = nullptr;                       /* tile counter of the compaction */
    long long *h_kept = nullptr;                         /* pinned: kept letters of the last compaction */
    cudaEvent_t k_done = nullptr;                        /* the last skip call's work that reads k_* has been issued before it */
    cudaEvent_t k_t0 = nullptr, k_t1 = nullptr;          /* kernel timing of the compaction and the remap */
    /* workspace of acb_lookup_host (keys and offsets go to w_hay / w_off) */
    int32_t *w_lk = nullptr; size_t w_lk_cap = 0;        /* key_id[n] then prefix[n] */
    /* dictionary view of the select calls (acb_table_upload_key_ranges), uploaded on first use */
    int32_t *d_order = nullptr, *d_lo = nullptr, *d_cnt = nullptr, *d_child_ptr = nullptr, *d_child = nullptr;
    /* workspace of the select calls */
    uint8_t *w_scan = nullptr; size_t w_scan_cap = 0;    /* the offsets' prefix sum */
    long long *w_sel_off = nullptr; size_t w_sel_off_cap = 0;   /* acb_select_host: out offsets[n+1] then the total */
    int32_t *w_sel_id = nullptr; size_t w_sel_id_cap = 0;       /* acb_select_host: key ids */
    /* workspace of the leftmost-longest selection (acb_leftmost_longest_device), sized by the full record count */
    Scratch l_buf;                                       /* sort keys, sorted records, candidates, flags, successors, cub scratch */
    unsigned long long *l_ctr = nullptr;                 /* [0] candidates, [1] chain tile counter, [2] chosen count (host route) */
    acb_match *l_out = nullptr; size_t l_out_cap = 0;    /* acb_scan_host_leftmost: the chosen records */
    cudaEvent_t l_ev[6] = {};                            /* kernel timing of its stages */
    /* workspace of the leftmost-longest replacement (acb_replace_device), sized by the chosen records' capacity */
    Scratch r_buf;                                       /* shifts, per-record positions, cub scratch; its event also guards r_ts */
    long long *r_ts = nullptr; size_t r_ts_cap = 0;      /* the last record that starts at or before each tile start */
    uint8_t *r_out = nullptr; size_t r_out_cap = 0;      /* acb_replace_host: the output bytes */
    long long *r_off = nullptr; size_t r_off_cap = 0;    /* acb_replace_host: output offsets[n+1] then the total */
    cudaEvent_t r_ev[4] = {};                            /* kernel timing of the offsets pass and the write pass */
    /* workspace of the whole-word filter (acb_word_filter_device), sized by the record count */
    Scratch ww_buf;                                      /* flags, positions, the record count, cub scratch */
    uint32_t *ww_bits = nullptr; size_t ww_bits_cap = 0; /* the host routes: their word bitmap */
    acb_match *ww_out = nullptr; size_t ww_out_cap = 0;  /* the host routes: the whole-word records */
    cudaEvent_t ww_ev[2] = {};                           /* kernel timing of the filter */
    int cta_limit = 0;                       /* acb_table_set_cta_limit: 0, or the SMs the launches act as if the device had */
    /* case folding: every scan reads a folded copy of the text.  fold: 0 none, 1 ASCII (acb_table_upload_folded), 2 a
     * letter map (acb_table_upload_folded_map), whose device tables are d_fold_map, fold_map16 16-byte blocks */
    int fold = 0;
    uint4 *d_fold_map = nullptr; int fold_map16 = 0;
    int32_t n_rep = 0;                                   /* ids the alias CSR covers: the trie's n_keys */
    int64_t n_alias = 0;                                 /* alias ids; 0: no key set member has a case variant */
    int32_t *d_alias_ptr = nullptr, *d_alias_ids = nullptr;   /* per representative id, its other ids, ascending */
    Scratch f_buf;                                       /* acb_scan_device: the folded copy of the batch */
    Scratch x_buf;                                       /* the alias expansion: per-record positions, cub scratch */
    acb_match *x_out = nullptr; size_t x_out_cap = 0;    /* the host routes: the expanded records */
    cudaEvent_t f_ev[4] = {};                            /* kernel timing of the fold and of the expansion */
};

/* The calling thread's current device, saved when an exported entry point starts and made current again on every return
 * path.  Entry points switch to the device of their table, stream batch or replacer (cudaSetDevice); without this the
 * caller's next CUDA work -- its own allocations, or the next call that reads the current device -- would land there.
 * An entry point that calls another one after switching gets the switched device back from it. */
class DeviceRestore {
    int prev_ = -1;
public:
    DeviceRestore() { if (cudaGetDevice(&prev_) != cudaSuccess) prev_ = -1; }
    ~DeviceRestore() {
        int cur = -1;
        if (prev_ >= 0 && cudaGetDevice(&cur) == cudaSuccess && cur != prev_) cudaSetDevice(prev_);
    }
    DeviceRestore(const DeviceRestore &) = delete;
    DeviceRestore &operator=(const DeviceRestore &) = delete;
};

extern "C" int acb_device_count(int32_t *n) {
    int c = 0;
    cudaError_t e = cudaGetDeviceCount(&c);
    if (e != cudaSuccess) { acb_set_error("cudaGetDeviceCount: %s", cudaGetErrorString(e)); if (n) *n = 0; return ACB_ECUDA; }
    if (n) *n = c;
    return ACB_OK;
}

template <typename T>
static int upload(T **dst, const T *src, size_t n, long long &acc) {
    size_t bytes = std::max<size_t>(n, 1) * sizeof(T);
    bytes = (bytes + 15) & ~(size_t)15;
    CUDA_TRY(cudaMalloc(reinterpret_cast<void **>(dst), bytes));
    CUDA_TRY(cudaMemset(*dst, 0, bytes));
    if (n) CUDA_TRY(cudaMemcpy(*dst, src, n * sizeof(T), cudaMemcpyHostToDevice));
    acc += (long long)bytes;
    return ACB_OK;
}

extern "C" void acb_table_free(acb_table *tb) {
    DeviceRestore keep_device;
    if (!tb) return;
    cudaSetDevice(tb->device);
    cudaFree(tb->d_lfail); cudaFree(tb->d_cls); cudaFree(tb->d_goto); cudaFree(tb->d_fail); cudaFree(tb->d_keyof);
    cudaFree(tb->d_outptr); cudaFree(tb->d_outidx); cudaFree(tb->d_keylen); cudaFree(tb->d_bm1); cudaFree(tb->d_bm3); cudaFree(tb->d_anchors);
    tb->sort_buf.release(); cudaFree(tb->d_work); cudaFree(tb->d_cand); cudaFree(tb->d_long_final); cudaFree(tb->w_hay); cudaFree(tb->w_off); cudaFree(tb->w_out); cudaFree(tb->w_count);
    if (tb->h_count) cudaFreeHost(tb->h_count);
    if (tb->h_out) cudaFreeHost(tb->h_out);
    if (tb->ev0) cudaEventDestroy(tb->ev0);
    if (tb->ev1) cudaEventDestroy(tb->ev1);
    if (tb->stream) cudaStreamDestroy(tb->stream);
    if (tb->s_copy) cudaStreamDestroy(tb->s_copy);
    if (tb->s_sort) cudaStreamDestroy(tb->s_sort);
    for (cudaEvent_t e : tb->ev_h2d) cudaEventDestroy(e);
    for (cudaEvent_t e : tb->ev_scan) cudaEventDestroy(e);
    if (tb->h_counts) cudaFreeHost(tb->h_counts);
    cudaFree(tb->k_buf); cudaFree(tb->k_mask); cudaFree(tb->k_gpre); cudaFree(tb->k_tile_pre); cudaFree(tb->k_status);
    cudaFree(tb->k_coff); cudaFree(tb->k_set); cudaFree(tb->k_ctr);
    cudaFree(tb->w_lk);
    cudaFree(tb->d_order); cudaFree(tb->d_lo); cudaFree(tb->d_cnt); cudaFree(tb->d_child_ptr); cudaFree(tb->d_child);
    cudaFree(tb->w_scan); cudaFree(tb->w_sel_off); cudaFree(tb->w_sel_id);
    tb->l_buf.release(); cudaFree(tb->l_ctr); cudaFree(tb->l_out);
    for (cudaEvent_t e : tb->l_ev) if (e) cudaEventDestroy(e);
    tb->r_buf.release(); cudaFree(tb->r_ts); cudaFree(tb->r_out); cudaFree(tb->r_off);
    for (cudaEvent_t e : tb->r_ev) if (e) cudaEventDestroy(e);
    tb->ww_buf.release(); cudaFree(tb->ww_bits); cudaFree(tb->ww_out);
    for (cudaEvent_t e : tb->ww_ev) if (e) cudaEventDestroy(e);
    if (tb->h_kept) cudaFreeHost(tb->h_kept);
    if (tb->k_done) cudaEventDestroy(tb->k_done);
    if (tb->k_t0) cudaEventDestroy(tb->k_t0);
    if (tb->k_t1) cudaEventDestroy(tb->k_t1);
    cudaFree(tb->d_alias_ptr); cudaFree(tb->d_alias_ids); tb->f_buf.release(); tb->x_buf.release(); cudaFree(tb->x_out);
    cudaFree(tb->d_fold_map);
    for (cudaEvent_t e : tb->f_ev) if (e) cudaEventDestroy(e);
    delete tb;
}

extern "C" int acb_table_upload(const acb_trie *t, int device, acb_table **out) {
    DeviceRestore keep_device;
    if (!t || !out) { acb_set_error("bad argument"); return ACB_EINVAL; }
    *out = nullptr;
    acb_flat_view f;
    int rc = acb_trie_flat_view(t, &f);
    if (rc != ACB_OK) return rc;
    if (f.n_states > kIdMask) { acb_set_error("too many states for the device table (%d)", f.n_states); return ACB_ERANGE; }
    int ndev = 0;
    CUDA_TRY(cudaGetDeviceCount(&ndev));
    if (device < 0 || device >= ndev) { acb_set_error("no such CUDA device %d (have %d)", device, ndev); return ACB_ECUDA; }
    CUDA_TRY(cudaSetDevice(device));
    acb_table *tb = new (std::nothrow) acb_table();
    if (!tb) { acb_set_error("out of memory"); return ACB_ENOMEM; }
    tb->device = device;
    cudaDeviceProp prop;
    rc = ACB_OK;
    do {
        if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) { acb_set_error("cudaGetDeviceProperties failed"); rc = ACB_ECUDA; break; }
        tb->sm_count = prop.multiProcessorCount;
        tb->S = f.n_states; tb->K = f.n_classes; tb->L = f.letter_bytes; tb->n_keys = f.n_keys;
        tb->gram = f.gram_bytes; tb->stride = f.stride; tb->log1 = f.log2_bits1; tb->log3 = f.log2_bits3; tb->logA = f.log2_anchor_slots; tb->filter_flags = f.filter_flags; tb->log2b = f.log2_bits2;
        tb->min_key_bytes = f.min_key_bytes; tb->max_key_bytes = f.max_key_bytes;
        acb_hash_multipliers(tb->gram, 1, tb->mul1);
        acb_hash_multipliers(tb->gram, 2, tb->mul2);
        try {
            tb->key_len.assign(f.key_len, f.key_len + f.n_keys);
        } catch (const std::exception &) {                   /* nothing may cross the C ABI */
            acb_set_error("out of host memory while staging the tables");
            rc = ACB_ENOMEM;
            break;
        }
        if ((rc = upload(&tb->d_cls, f.byte_class, 256, tb->dev_bytes))) break;
        if ((rc = upload(&tb->d_goto, f.goto_cm, (size_t)f.n_classes * f.n_states, tb->dev_bytes))) break;
        if ((rc = upload(&tb->d_fail, f.fail, (size_t)f.n_states, tb->dev_bytes))) break;
        if ((rc = upload(&tb->d_lfail, f.letter_fail, (size_t)f.n_states, tb->dev_bytes))) break;
        if ((rc = upload(&tb->d_keyof, f.key_of, (size_t)f.n_states, tb->dev_bytes))) break;
        {   /* goto entries get a flag bit when the child ends a key, saving a key_of lookup per step: set on the device,
               in place (no second host copy of a table that can be gigabytes) */
            const size_t n = (size_t)f.n_classes * f.n_states;
            acb_flag_goto_kernel<<<(unsigned)std::min<size_t>((n + 255) / 256, 1u << 20), 256>>>(tb->d_goto, tb->d_keyof, n);
            if (cudaDeviceSynchronize() != cudaSuccess) { acb_set_error("flagging the goto table failed: %s", cudaGetErrorString(cudaGetLastError())); rc = ACB_ECUDA; break; }
        }
        if ((rc = upload(&tb->d_outptr, f.out_ptr, (size_t)f.n_states + 1, tb->dev_bytes))) break;
        if ((rc = upload(&tb->d_outidx, f.out_idx, (size_t)f.out_ptr[f.n_states], tb->dev_bytes))) break;
        if ((rc = upload(&tb->d_keylen, f.key_len, (size_t)f.n_keys, tb->dev_bytes))) break;
        if ((rc = upload(&tb->d_bm1, f.bitmap1, ((size_t)1 << (f.log2_bits1 - 5)) + (f.log2_bits2 ? (size_t)1 << (f.log2_bits2 - 5) : 0), tb->dev_bytes))) break;
        if ((rc = upload(&tb->d_bm3, f.bitmap3, f.log2_bits3 ? ((size_t)1 << (f.log2_bits3 - 5)) : 1, tb->dev_bytes))) break;
        if ((rc = upload(&tb->d_anchors, f.anchors, (size_t)8 << f.log2_anchor_slots, tb->dev_bytes))) break;
        unsigned int zero[4] = {0, 0, 0, 0};   /* work counters, re-armed by the kernels themselves */
        if ((rc = upload(&tb->d_work, zero, 4, tb->dev_bytes))) break;
    } while (0);
    if (rc != ACB_OK) { acb_table_free(tb); return rc; }
    *out = tb;
    return ACB_OK;
}

extern "C" int64_t acb_table_device_bytes(const acb_table *tb) { return tb ? tb->dev_bytes : 0; }

/* the SMs a launch spreads over: one persistent CTA each, and the bound of the grid-stride loops */
static long long grid_sms(const acb_table *tb) {
    return tb->cta_limit > 0 ? std::min(tb->cta_limit, tb->sm_count) : tb->sm_count;
}

/* the grid of a grid-stride launch over `items`: a block per `threads` of them, at most 16 per SM */
static unsigned blocks(const acb_table *tb, long long items, int threads = 256) {
    return (unsigned)std::min<long long>((items + threads - 1) / threads, grid_sms(tb) * 16);
}

/* f(std::integral_constant<int, L>()) for the letter width L (1, 2 or 4), so f can launch the kernel templated on it */
template <class F>
static void with_width(int L, F &&f) {
    if (L == 1) f(std::integral_constant<int, 1>());
    else if (L == 2) f(std::integral_constant<int, 2>());
    else f(std::integral_constant<int, 4>());
}

/* haystack h of a batch starts at byte off[h], or at h * stride without offsets; it ends where haystack h + 1 starts */
static __device__ __forceinline__ long long hay_start(const long long *off, long long stride, long long h) {
    return off ? __ldg(off + h) : h * stride;
}

extern "C" int acb_table_set_cta_limit(acb_table *tb, int32_t n) {
    if (!tb || n < 0) { acb_set_error("bad argument"); return ACB_EINVAL; }
    tb->cta_limit = n;
    return ACB_OK;
}

extern "C" int acb_scan_geometry(int pair, int32_t *out, int32_t n) {
    if (!out || n < 6) { acb_set_error("bad argument"); return ACB_EINVAL; }
    const int32_t g[2][6] = {{kSliceBytes, kTileBytes, kStages, kConsumers, kClaimDepth, kLook},
                             {kSliceBytes, kPairTileBytes, kPairStages, kPairConsumers, kClaimDepth, kLook}};
    memcpy(out, g[pair != 0], sizeof(g[0]));
    return ACB_OK;
}

/* the launch shape of a filter scan of one segment (<= kSegBytes): tiles of the kernel's ring, one CTA per SM */
extern "C" int acb_table_scan_grid(const acb_table *tb, int64_t total_bytes, int32_t *grid, int64_t *n_tiles) {
    if (!tb || !grid || !n_tiles || total_bytes < 0 || total_bytes > kSegBytes) { acb_set_error("bad argument"); return ACB_EINVAL; }
    const long long tile_bytes = (tb->filter_flags & ACB_FILTER_PAIR) ? kPairTileBytes : kTileBytes;
    *n_tiles = (total_bytes + tile_bytes - 1) / tile_bytes;
    *grid = (int32_t)std::min<long long>(grid_sms(tb), *n_tiles);
    return ACB_OK;
}
extern "C" int64_t acb_launch_count(void) { return g_launches.load(); }
extern "C" int acb_set_kernel_timing(int enabled) { g_timing.store(enabled ? 1 : 0); return ACB_OK; }
extern "C" float acb_last_kernel_ms(void) { return g_last_ms; }

/* ----------------------------------------------------- shared host checks */

/* after a launch (acb_launch_count): its error, naming the kernel, or n more launches; n > 1 counts a group once */
static int launched(const char *what, int n = 1) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { acb_set_error("%s launch failed: %s", what, cudaGetErrorString(e)); return ACB_ECUDA; }
    g_launches.fetch_add(n);
    return ACB_OK;
}

/* kernel timing (acb_set_kernel_timing): event *ev recorded on s, created on first use; nothing while timing is off */
static int timing_mark(cudaEvent_t *ev, cudaStream_t s) {
    if (!g_timing.load()) return ACB_OK;
    if (!*ev) CUDA_TRY(cudaEventCreate(ev));
    CUDA_TRY(cudaEventRecord(*ev, s));
    return ACB_OK;
}

/* *ms = the time from mark a to mark b, waiting for b; *ms untouched while timing is off */
static int timing_ms(cudaEvent_t a, cudaEvent_t b, float *ms) {
    if (!g_timing.load()) return ACB_OK;
    CUDA_TRY(cudaEventSynchronize(b));
    CUDA_TRY(cudaEventElapsedTime(ms, a, b));
    return ACB_OK;
}

/* a fixed-stride batch: stride >= min_stride (0 or 1), a multiple of the letter width, and n * stride == total, checked
 * without overflowing n * stride */
static int check_stride(int32_t L, int64_t total, int64_t n, int64_t stride, int64_t min_stride) {
    if (stride >= min_stride && stride % L == 0 && (stride == 0 ? total == 0 : n <= total / stride && n * stride == total)) return ACB_OK;
    acb_set_error("a fixed-stride batch needs stride_bytes >= %lld, a multiple of letter_bytes, and n*stride_bytes == total_bytes",
                  (long long)min_stride);
    return ACB_EINVAL;
}

/* a table uploaded by acb_table_upload_folded: refused by the entries that do not fold their text */
static int refuse_folded(const acb_table *tb, const char *what) {
    if (!tb || !tb->fold) return ACB_OK;
    acb_set_error("%s does not take a case-folded table", what);
    return ACB_EINVAL;
}

/* ------------------------------------------------------------- launching */

constexpr int kMaxDevices = 64;                              /* opt-in caches below are per device */

/* Opts the current device's kernels into `smem` bytes of dynamic shared memory once: `opted` is the largest size they were
 * set to so far (per instantiation and device) and only grows.  Check, set and store happen under one lock, so the cache
 * is never ahead of the attribute: two threads that opt in to sizes a < b at once otherwise can leave the cache at b and
 * the attribute at a, and every later launch that needs b fails.  The load before the lock keeps the common path free. */
template <class SetAll>
static int opt_in_smem(std::atomic<size_t> &opted, size_t smem, SetAll &&set_all) {
    if (opted.load(std::memory_order_acquire) >= smem) return ACB_OK;
    static std::mutex mu;
    std::lock_guard<std::mutex> lk(mu);
    if (opted.load(std::memory_order_relaxed) >= smem) return ACB_OK;
    int rc = set_all(smem);
    if (rc == ACB_OK) opted.store(smem, std::memory_order_release);
    return rc;
}

template <int NW, int STRIDE, int MODE>
static int launch_stream_m(const ScanParams &p, int grid, cudaStream_t s) {
    auto kern = acb_stream_kernel<NW, STRIDE, MODE>;
    const size_t smem = stream_smem(p.log1).total;
    static std::atomic<size_t> opted_dev[kMaxDevices];
    int dev = 0;
    CUDA_TRY(cudaGetDevice(&dev));                           /* the attribute belongs to the current device's context */
    int rc = opt_in_smem(opted_dev[dev % kMaxDevices], smem, [&](size_t n) {
        CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)n));
        return ACB_OK;
    });
    if (rc != ACB_OK) return rc;
    kern<<<grid, kFThreads, smem, s>>>(p);
    return launched("stream kernel");
}

static int launch_pair(const ScanParams &p, int grid, cudaStream_t s) {
    const size_t smem = pair_smem(p.log1, p.log2b).total;
    static std::atomic<size_t> opted_dev[kMaxDevices];
    int dev = 0;
    CUDA_TRY(cudaGetDevice(&dev));
    int rc = opt_in_smem(opted_dev[dev % kMaxDevices], smem, [](size_t n) {
        CUDA_TRY(cudaFuncSetAttribute(acb_pair_kernel<17>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)n));
        CUDA_TRY(cudaFuncSetAttribute(acb_pair_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)n));
        return ACB_OK;
    });
    if (rc != ACB_OK) return rc;
    if (p.log2b == 17) acb_pair_kernel<17><<<grid, kPairThreads, smem, s>>>(p);      /* the 2^20-bit level 1 of 10 k keys and more */
    else acb_pair_kernel<0><<<grid, kPairThreads, smem, s>>>(p);
    return launched("pair kernel");
}

/* the placement mode follows from the table's filter_flags */
template <int NW, int STRIDE>
static int launch_stream_t(const ScanParams &p, int flags, int grid, cudaStream_t s) {
    if (flags & ACB_FILTER_PAIR) {
        if (NW != 1 || STRIDE != 1 || p.gram != 4 || p.L != 1 || p.log2b < 13 || p.log2b > 19) { acb_set_error("PAIR filter needs gram 4, stride 1, 1-byte letters and a level 2"); return ACB_EINVAL; }
        return launch_pair(p, grid, s);
    }
    if (flags & ACB_FILTER_WIDE) {
        if (p.gram != 4 * NW) { acb_set_error("WIDE filter with gram %d", p.gram); return ACB_EINVAL; }
        return launch_stream_m<NW, STRIDE, kModeWide>(p, grid, s);
    }
    return launch_stream_m<NW, STRIDE, kModeNarrow>(p, grid, s);
}

template <int NW>
static int launch_stream_s(const ScanParams &p, int flags, int stride, int grid, cudaStream_t s) {
    switch (stride) {
        case 1:  return launch_stream_t<NW, 1>(p, flags, grid, s);
        case 2:  return launch_stream_t<NW, 2>(p, flags, grid, s);
        case 4:  return launch_stream_t<NW, 4>(p, flags, grid, s);
        case 8:  return launch_stream_t<NW, 8>(p, flags, grid, s);
        case 16: return launch_stream_t<NW, 16>(p, flags, grid, s);
    }
    acb_set_error("unsupported filter stride %d", stride);
    return ACB_EINVAL;
}

static int launch_stream(const ScanParams &p, int flags, int stride, int grid, cudaStream_t s) {
    switch ((p.gram + 3) / 4) {
        case 1: return launch_stream_s<1>(p, flags, stride, grid, s);
        case 2: return launch_stream_s<2>(p, flags, stride, grid, s);
        case 3: return launch_stream_s<3>(p, flags, stride, grid, s);
        case 4: return launch_stream_s<4>(p, flags, stride, grid, s);
    }
    acb_set_error("unsupported gram length %d", p.gram);
    return ACB_EINVAL;
}

/* the stream kernel over the start positions [begin, end) of the flat buffer (begin a multiple of 32), one launch per
 * <= 2 GiB segment.  Text after `end` is read as far as a key can reach, never interpreted as a start position. */
static int launch_filter_range(acb_table *tb, ScanParams &p, long long begin, long long end, cudaStream_t s) {
    if (!(tb->filter_flags & ACB_FILTER_PAIR) && !tb->d_cand) {    /* room for every byte of a slice per consumer warp: never overflows */
        CUDA_TRY(cudaMalloc(reinterpret_cast<void **>(&tb->d_cand), (size_t)tb->sm_count * kConsumers * kWarpCand * sizeof(uint2)));
        tb->dev_bytes += (long long)tb->sm_count * kConsumers * kWarpCand * (long long)sizeof(uint2);
    }
    p.cand = tb->d_cand;
    for (long long seg = begin; seg < end; seg += kSegBytes) {
        p.seg_begin = seg;
        p.seg_end = std::min<long long>(seg + kSegBytes, end);
        int32_t grid = 0;
        int64_t n_tiles = 0;
        int rc = acb_table_scan_grid(tb, p.seg_end - p.seg_begin, &grid, &n_tiles);
        if (rc != ACB_OK) return rc;
        p.n_tiles = (unsigned int)n_tiles;
        rc = launch_stream(p, tb->filter_flags, tb->stride, grid, s);
        if (rc != ACB_OK) return rc;
    }
    return ACB_OK;
}

static void fill_params(const acb_table *tb, ScanParams &p, const uint8_t *d_hay, int64_t total_bytes, const int64_t *d_offsets,
                        int64_t n_hay, int64_t stride_bytes, acb_match *d_out, int64_t cap, int64_t *d_count) {
    memset(&p, 0, sizeof(p));
    p.hay = d_hay; p.total = total_bytes; p.offsets = reinterpret_cast<const long long *>(d_offsets);
    p.n_hay = n_hay; p.stride_bytes = stride_bytes;
    p.cls = tb->d_cls; p.gto = tb->d_goto; p.fail = tb->d_fail; p.letter_fail = tb->d_lfail; p.key_of = tb->d_keyof;
    p.out_ptr = tb->d_outptr; p.out_idx = tb->d_outidx; p.key_len = tb->d_keylen;
    p.S = tb->S; p.L = tb->L; p.gram = tb->gram; p.max_key_bytes = tb->max_key_bytes;
    p.bm1 = tb->d_bm1; p.bm3 = tb->d_bm3; p.anchors = reinterpret_cast<const uint4 *>(tb->d_anchors);
    p.log1 = tb->log1; p.log3 = tb->log3; p.logA = tb->logA; p.log2b = tb->log2b;
    memcpy(p.mul1, tb->mul1, sizeof(p.mul1));
    memcpy(p.mul2, tb->mul2, sizeof(p.mul2));
    p.out = d_out; p.cap = cap; p.count = reinterpret_cast<unsigned long long *>(d_count);
    p.work_ctr = tb->d_work;
    p.stride_shift = -1;
    if (!d_offsets) for (int b = 0; b < 62; b++) if ((1LL << b) == stride_bytes) p.stride_shift = b;
    p.letter_shift = tb->L == 4 ? 2 : (tb->L == 2 ? 1 : 0);
}

/* ------------------------------------------------------------- ASCII case folding */
/* A folded table's scans read the text with every ASCII capital (letter value 0x41..0x5A) made small (+0x20); nothing
 * else changes, so positions and lengths are those of the text.  1-byte letters: four per 32-bit word, tested together
 * (SWAR); 4-byte letters: the whole letter value is compared, so U+0141 or U+1F641 never fold. */
namespace {
thread_local float g_fold_ms[2] = {};                      /* kernel timing: fold, alias expansion */

/* the bytes of x with 0x41..0x5A made small: h + 0x3f carries into bit 7 iff h >= 0x41, h + 0x25 iff h >= 0x5b (h <= 0x7f,
 * so no byte carries into the next); a byte with bit 7 set is never a capital */
__device__ __forceinline__ uint32_t fold_bytes(uint32_t x) {
    const uint32_t h = x & 0x7f7f7f7fu;
    const uint32_t upper = (h + 0x3f3f3f3fu) & ~(h + 0x25252525u) & ~x & 0x80808080u;
    return x | upper >> 2;
}

template <int L>
__device__ __forceinline__ uint32_t fold_word(uint32_t v) {
    return L == 1 ? fold_bytes(v) : (v - 0x41u < 26u ? v + 0x20u : v);
}

template <int L>
__device__ __forceinline__ uint4 fold_block(uint4 v) {
    return make_uint4(fold_word<L>(v.x), fold_word<L>(v.y), fold_word<L>(v.z), fold_word<L>(v.w));
}

/* out = the n16 16-byte blocks of in folded, then `tail` (< 16, a multiple of L) more bytes; in == out is allowed.  Each
 * thread keeps four blocks in flight per turn of the grid-stride loop. */
template <int L>
__global__ void __launch_bounds__(256) acb_fold_kernel(const uint4 *in, uint4 *out, long long n16, int tail) {
    const long long step = (long long)gridDim.x * blockDim.x;
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    for (; i + 3 * step < n16; i += 4 * step) {
        uint4 v[4];
#pragma unroll
        for (int k = 0; k < 4; k++) v[k] = in[i + k * step];
#pragma unroll
        for (int k = 0; k < 4; k++) out[i + k * step] = fold_block<L>(v[k]);
    }
    for (; i < n16; i += step) out[i] = fold_block<L>(in[i]);
    if (blockIdx.x == 0 && (int)threadIdx.x * L < tail) {
        if (L == 1) {
            const uint8_t b = reinterpret_cast<const uint8_t *>(in + n16)[threadIdx.x];
            reinterpret_cast<uint8_t *>(out + n16)[threadIdx.x] = (uint8_t)(b - 0x41u < 26u ? b + 0x20u : b);
        } else {
            reinterpret_cast<uint32_t *>(out + n16)[threadIdx.x] = fold_word<L>(reinterpret_cast<const uint32_t *>(in + n16)[threadIdx.x]);
        }
    }
}

/* ------------------------------------------------------------- mapped case folding (acb_table_upload_folded_map) */
/* A letter map folds each letter alone: 1-byte letters through a 256-byte table; 4-byte letters below 0x110000 through
 * two levels -- page[v >> 8] picks one of the 256-entry blocks, whose entry is the drop (v - folded v), block 0 all zero
 * -- and letters from 0x110000 up (not code points) stay as they are.  The device buffer holds the blocks, then the
 * 4352 page indices; every CTA stages it in shared memory before it reads the text. */
constexpr int kFoldPages = 0x110000 >> 8;
constexpr int kFoldMaxBlocks = (48 * 1024 - kFoldPages) / 1024;   /* the tables fit the 48 KiB a launch gets without opt-in */

template <int L>
__device__ __forceinline__ uint32_t map_word(uint32_t v, const uint32_t *drop, const uint8_t *page) {
    if (L == 1) {
        const uint8_t *m = page;
        return m[v & 255] | (uint32_t)m[(v >> 8) & 255] << 8 | (uint32_t)m[(v >> 16) & 255] << 16 | (uint32_t)m[v >> 24] << 24;
    }
    return v < 0x110000u ? v - drop[(uint32_t)page[v >> 8] << 8 | (v & 255)] : v;
}

template <int L>
__device__ __forceinline__ uint4 map_block(uint4 v, const uint32_t *drop, const uint8_t *page) {
    return make_uint4(map_word<L>(v.x, drop, page), map_word<L>(v.y, drop, page), map_word<L>(v.z, drop, page),
                      map_word<L>(v.w, drop, page));
}

/* acb_fold_kernel's loop with the letter map `map` (map16 16-byte blocks) staged in shared memory; in == out is allowed */
template <int L>
__global__ void __launch_bounds__(256) acb_map_fold_kernel(const uint4 *in, uint4 *out, long long n16, int tail,
                                                          const uint4 *__restrict__ map, int map16) {
    extern __shared__ uint4 s_map[];
    for (int j = threadIdx.x; j < map16; j += blockDim.x) s_map[j] = map[j];
    __syncthreads();
    const uint32_t *drop = reinterpret_cast<const uint32_t *>(s_map);
    const uint8_t *page = L == 1 ? reinterpret_cast<const uint8_t *>(s_map)
                                 : reinterpret_cast<const uint8_t *>(s_map + map16) - kFoldPages;
    const long long step = (long long)gridDim.x * blockDim.x;
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    for (; i + 3 * step < n16; i += 4 * step) {
        uint4 v[4];
#pragma unroll
        for (int k = 0; k < 4; k++) v[k] = in[i + k * step];
#pragma unroll
        for (int k = 0; k < 4; k++) out[i + k * step] = map_block<L>(v[k], drop, page);
    }
    for (; i < n16; i += step) out[i] = map_block<L>(in[i], drop, page);
    if (blockIdx.x == 0 && (int)threadIdx.x * L < tail) {
        if (L == 1) {
            const uint8_t b = reinterpret_cast<const uint8_t *>(in + n16)[threadIdx.x];
            reinterpret_cast<uint8_t *>(out + n16)[threadIdx.x] = page[b];
        } else {
            reinterpret_cast<uint32_t *>(out + n16)[threadIdx.x] = map_word<L>(reinterpret_cast<const uint32_t *>(in + n16)[threadIdx.x], drop, page);
        }
    }
}
} // namespace

/* the fold of `bytes` bytes at in (16-byte aligned) to out (16-byte aligned, may be in), on s: one launch */
static int fold_text(const acb_table *tb, const uint8_t *in, uint8_t *out, long long bytes, cudaStream_t s) {
    const long long n16 = bytes / 16;
    const int tail = (int)(bytes % 16);
    auto *i4 = reinterpret_cast<const uint4 *>(in);
    auto *o4 = reinterpret_cast<uint4 *>(out);
    if (tb->fold == 2) {        /* every CTA stages the map: four per SM keep enough loads in flight and stage it less often */
        const unsigned grid = (unsigned)std::max<long long>(std::min<long long>(blocks(tb, n16), grid_sms(tb) * 4), 1);
        const size_t smem = (size_t)tb->fold_map16 * 16;
        if (tb->L == 1) acb_map_fold_kernel<1><<<grid, 256, smem, s>>>(i4, o4, n16, tail, tb->d_fold_map, tb->fold_map16);
        else acb_map_fold_kernel<4><<<grid, 256, smem, s>>>(i4, o4, n16, tail, tb->d_fold_map, tb->fold_map16);
        return launched("case fold");
    }
    const unsigned grid = std::max(blocks(tb, n16), 1u);
    if (tb->L == 1) acb_fold_kernel<1><<<grid, 256, 0, s>>>(i4, o4, n16, tail);
    else acb_fold_kernel<4><<<grid, 256, 0, s>>>(i4, o4, n16, tail);
    return launched("case fold");
}

extern "C" int acb_table_upload_folded(const acb_trie *t, int device, const int32_t *alias_ptr, const int32_t *alias_ids,
                                       int64_t n_alias, acb_table **out) {
    DeviceRestore keep_device;
    if (!t || !out || n_alias < 0 || (n_alias && (!alias_ptr || !alias_ids))) { acb_set_error("bad argument"); return ACB_EINVAL; }
    *out = nullptr;
    acb_flat_view f;
    int rc = acb_trie_flat_view(t, &f);
    if (rc != ACB_OK) return rc;
    if (f.letter_bytes != 1 && f.letter_bytes != 4) { acb_set_error("case folding takes 1- or 4-byte letters, not %d", f.letter_bytes); return ACB_EINVAL; }
    /* the alias lists: alias_ptr[0 .. n_keys] from 0 to n_alias, each list ascending above its representative, which is a
     * live key of the trie */
    int32_t max_id = f.n_keys - 1;
    if (alias_ptr) {
        bool ok = alias_ptr[0] == 0 && alias_ptr[f.n_keys] == n_alias;
        for (int32_t k = 0; ok && k < f.n_keys; k++) {
            ok = alias_ptr[k + 1] >= alias_ptr[k] && (alias_ptr[k + 1] == alias_ptr[k] || f.key_len[k] > 0);
            for (int32_t j = alias_ptr[k]; ok && j < alias_ptr[k + 1]; j++) {
                ok = alias_ids[j] > (j == alias_ptr[k] ? k : alias_ids[j - 1]) && alias_ids[j] < 0x7fffffff;
                if (ok) max_id = std::max(max_id, alias_ids[j]);
            }
        }
        if (!ok) {
            acb_set_error("alias lists must run from 0 to n_alias over n_keys + 1 offsets, each ascending above its live key id");
            return ACB_EINVAL;
        }
    }
    if ((rc = acb_table_upload(t, device, out))) return rc;
    acb_table *tb = *out;
    tb->fold = 1;
    tb->n_rep = f.n_keys;
    tb->n_alias = n_alias;
    do {
        if (!n_alias) break;
        if (cudaSetDevice(device) != cudaSuccess) {        /* acb_table_upload gave the caller's device back */
            acb_set_error("cudaSetDevice(%d) failed", device);
            rc = ACB_ECUDA;
            break;
        }
        try {                                              /* an alias has its representative's length */
            tb->key_len.resize((size_t)max_id + 1, 0);
            for (int32_t k = 0; k < f.n_keys; k++)
                for (int32_t j = alias_ptr[k]; j < alias_ptr[k + 1]; j++) tb->key_len[alias_ids[j]] = f.key_len[k];
        } catch (const std::exception &) {
            acb_set_error("out of host memory while staging the tables");
            rc = ACB_ENOMEM;
            break;
        }
        cudaFree(tb->d_keylen);                            /* replaced by the longer list, as upload() sized it */
        tb->d_keylen = nullptr;
        tb->dev_bytes -= (long long)(((size_t)std::max(f.n_keys, 1) * sizeof(int32_t) + 15) & ~(size_t)15);
        tb->n_keys = max_id + 1;
        if ((rc = upload(&tb->d_keylen, tb->key_len.data(), tb->key_len.size(), tb->dev_bytes))) break;
        if ((rc = upload(&tb->d_alias_ptr, alias_ptr, (size_t)f.n_keys + 1, tb->dev_bytes))) break;
        rc = upload(&tb->d_alias_ids, alias_ids, (size_t)n_alias, tb->dev_bytes);
    } while (0);
    if (rc != ACB_OK) { acb_table_free(tb); *out = nullptr; }
    return rc;
}

extern "C" int acb_table_upload_folded_map(const acb_trie *t, int device, const int32_t *alias_ptr, const int32_t *alias_ids,
                                           int64_t n_alias, const uint32_t *map_from, const uint32_t *map_to, int64_t n_map,
                                           acb_table **out) {
    DeviceRestore keep_device;
    if (!t || !out || n_map < 0 || (n_map && (!map_from || !map_to))) { acb_set_error("bad argument"); return ACB_EINVAL; }
    *out = nullptr;
    acb_flat_view f;
    int rc = acb_trie_flat_view(t, &f);
    if (rc != ACB_OK) return rc;
    /* the map: from strictly ascending, each to below its from and not itself mapped (a fold applied twice changes nothing),
     * every from a code point; a 1-byte trie reads the entries below 256, which must stay there */
    bool ok = true;
    for (int64_t j = 0; ok && j < n_map; j++)
        ok = (j == 0 || map_from[j] > map_from[j - 1]) && map_to[j] < map_from[j] && map_from[j] < 0x110000u &&
             !std::binary_search(map_from, map_from + n_map, map_to[j]) && (f.letter_bytes != 1 || map_from[j] >= 256 || map_to[j] < 256);
    if (!ok) {
        acb_set_error("a letter map needs ascending code points, each mapped below itself to a letter the map leaves alone "
                      "(below 256 for a 1-byte trie)");
        return ACB_EINVAL;
    }
    std::vector<uint8_t> map;
    try {
        if (f.letter_bytes == 1) {
            map.resize(256);
            for (int b = 0; b < 256; b++) map[b] = (uint8_t)b;
            for (int64_t j = 0; j < n_map && map_from[j] < 256; j++) map[map_from[j]] = (uint8_t)map_to[j];
        } else {
            std::vector<uint8_t> page(kFoldPages, 0);
            int nb = 1;
            for (int64_t j = 0; j < n_map; j++)
                if (!page[map_from[j] >> 8]) page[map_from[j] >> 8] = (uint8_t)std::min(nb++, 255);
            if (nb > kFoldMaxBlocks) {
                acb_set_error("a letter map may change letters in at most %d blocks of 256 code points, not %d", kFoldMaxBlocks - 1, nb - 1);
                return ACB_EINVAL;
            }
            map.resize((size_t)nb * 1024 + kFoldPages, 0);
            auto *drop = reinterpret_cast<uint32_t *>(map.data());
            for (int64_t j = 0; j < n_map; j++)
                drop[(size_t)page[map_from[j] >> 8] << 8 | (map_from[j] & 255)] = map_from[j] - map_to[j];
            std::copy(page.begin(), page.end(), map.begin() + (size_t)nb * 1024);
        }
    } catch (const std::exception &) {
        acb_set_error("out of host memory while staging the tables");
        return ACB_ENOMEM;
    }
    if ((rc = acb_table_upload_folded(t, device, alias_ptr, alias_ids, n_alias, out))) return rc;
    acb_table *tb = *out;
    tb->fold = 2;
    tb->fold_map16 = (int)(map.size() / 16);
    if (cudaSetDevice(device) != cudaSuccess) {            /* acb_table_upload_folded gave the caller's device back */
        acb_set_error("cudaSetDevice(%d) failed", device);
        rc = ACB_ECUDA;
    } else {
        rc = upload(&tb->d_fold_map, reinterpret_cast<const uint4 *>(map.data()), map.size() / 16, tb->dev_bytes);
    }
    if (rc != ACB_OK) { acb_table_free(tb); *out = nullptr; }
    return rc;
}

extern "C" int acb_last_fold_ms(float *ms, int32_t n) {
    if (!ms || n < 0 || n > 2) { acb_set_error("bad argument"); return ACB_EINVAL; }
    for (int i = 0; i < n; i++) ms[i] = g_fold_ms[i];
    return ACB_OK;
}

static int scratch_take(Scratch &sc, size_t need, cudaStream_t s);
static int scratch_done(cudaEvent_t *done, cudaStream_t s);

/* an ACB_ALGO_LONG scan with no text or no keys launches nothing: haystack 0 ends in the state it starts in, and the
 * one-shot start state is consumed as by any other scan */
static void long_scan_without_launch(acb_table *tb) {
    tb->long_final_host = tb->long_init;
    tb->long_init = 0;
}

/* the scan launches of acb_scan_device over p, whose text a folded table's caller has already folded: timed by ev0 / ev1
 * into g_last_ms */
static int scan_text(acb_table *tb, ScanParams &p, int64_t total_bytes, int64_t n_hay, int algo, cudaStream_t s) {
    int rc;
    if ((rc = timing_mark(&tb->ev0, s))) return rc;
    if (algo == ACB_ALGO_FILTER) {
        if ((rc = launch_filter_range(tb, p, 0, total_bytes, s))) return rc;
    } else if (algo == ACB_ALGO_DFA) {
        long long spans = (total_bytes + kDfaSpan - 1) / kDfaSpan;
        long long grid = (spans + kDfaThreads - 1) / kDfaThreads;
        if (grid > 0x7fffffffLL) { acb_set_error("batch too large for one launch"); return ACB_ERANGE; }
        acb_dfa_kernel<<<(unsigned)grid, kDfaThreads, 0, s>>>(p);
        if ((rc = launched("DFA kernel"))) return rc;
    } else if (algo == ACB_ALGO_LONG) {
        if (!tb->d_long_final) CUDA_TRY(cudaMalloc(reinterpret_cast<void **>(&tb->d_long_final), sizeof(int32_t)));
        p.long_init = tb->long_init;
        p.long_final = tb->d_long_final;
        tb->long_init = 0;                                      /* one shot */
        tb->long_final_host = -1;                               /* the kernel writes the final state */
        long long grid = (n_hay + kDfaThreads - 1) / kDfaThreads;
        acb_long_kernel<<<(unsigned)grid, kDfaThreads, 0, s>>>(p);
        if ((rc = launched("iter_long kernel"))) return rc;
    } else {
        acb_set_error("unknown algo %d", algo);
        return ACB_EINVAL;
    }
    if ((rc = timing_mark(&tb->ev1, s))) return rc;
    return timing_ms(tb->ev0, tb->ev1, &g_last_ms);
}

/* the batch shapes a scan's records can describe (int32 hay_id and end_index): at most 2^31-1 haystacks, and a fixed
 * stride of at most 2^31-1 letters; checked before anything is launched */
static int check_scan_shape(const acb_table *tb, int64_t total_bytes, const int64_t *d_offsets, int64_t n_hay, int64_t stride_bytes) {
    if (n_hay > 0x7fffffffLL) { acb_set_error("more than 2^31-1 haystacks in one batch"); return ACB_ERANGE; }
    if (!d_offsets) {
        int rc = check_stride(tb->L, total_bytes, n_hay, stride_bytes, 1);
        if (rc != ACB_OK) return rc;
        if (stride_bytes / tb->L > 0x7fffffffLL) { acb_set_error("haystack longer than 2^31-1 letters"); return ACB_ERANGE; }
    }
    return ACB_OK;
}

extern "C" int acb_scan_device(acb_table *tb, const uint8_t *d_hay, int64_t total_bytes,
                               const int64_t *d_offsets, int64_t n_hay, int64_t stride_bytes,
                               acb_match *d_out, int64_t cap, int64_t *d_count, void *stream, int algo) {
    DeviceRestore keep_device;
    if (!tb || !d_count || total_bytes < 0 || n_hay < 0 || cap < 0 || (cap > 0 && !d_out)) { acb_set_error("bad argument"); return ACB_EINVAL; }
    if (algo == ACB_ALGO_LONG && refuse_folded(tb, "ACB_ALGO_LONG")) return ACB_EINVAL;
    if (int rc = check_scan_shape(tb, total_bytes, d_offsets, n_hay, stride_bytes)) return rc;
    if (total_bytes == 0 || n_hay == 0) {
        if (algo == ACB_ALGO_LONG) long_scan_without_launch(tb);
        return ACB_OK;
    }
    if (reinterpret_cast<uintptr_t>(d_hay) & 15) { acb_set_error("d_hay must be 16-byte aligned"); return ACB_EINVAL; }
    CUDA_TRY(cudaSetDevice(tb->device));
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);

    ScanParams p;
    fill_params(tb, p, d_hay, total_bytes, d_offsets, n_hay, stride_bytes, d_out, cap, d_count);

    if (algo == ACB_ALGO_AUTO) algo = ACB_ALGO_FILTER;
    if (tb->n_keys == 0) {                                  /* empty key set: nothing can match */
        if (algo == ACB_ALGO_LONG) long_scan_without_launch(tb);
        return ACB_OK;
    }
    int rc;
    if (tb->fold) {                                         /* the scan reads a folded copy; d_hay stays as the caller gave it */
        g_fold_ms[0] = 0.f;
        if ((rc = scratch_take(tb->f_buf, (size_t)total_bytes + 64, s)) || (rc = timing_mark(&tb->f_ev[0], s)) ||
            (rc = fold_text(tb, d_hay, static_cast<uint8_t *>(tb->f_buf.buf), total_bytes, s)) || (rc = timing_mark(&tb->f_ev[1], s)))
            return rc;
        p.hay = static_cast<const uint8_t *>(tb->f_buf.buf);
    }
    if ((rc = scan_text(tb, p, total_bytes, n_hay, algo, s))) return rc;
    if (tb->fold && ((rc = scratch_done(&tb->f_buf.done, s)) || (rc = timing_ms(tb->f_ev[0], tb->f_ev[1], &g_fold_ms[0])))) return rc;
    return ACB_OK;
}

extern "C" int acb_table_set_long_state(acb_table *tb, int32_t state) {
    if (!tb || state < 0 || state >= tb->S) { acb_set_error("not a state of this automaton"); return ACB_EINVAL; }
    tb->long_init = state;
    return ACB_OK;
}

extern "C" int acb_table_get_long_state(acb_table *tb, int32_t *state) {
    DeviceRestore keep_device;
    if (!tb || !state) { acb_set_error("bad argument"); return ACB_EINVAL; }
    *state = 0;
    if (tb->long_final_host >= 0) { *state = tb->long_final_host; return ACB_OK; }
    if (!tb->d_long_final) return ACB_OK;                    /* no ACB_ALGO_LONG scan yet */
    CUDA_TRY(cudaSetDevice(tb->device));
    CUDA_TRY(cudaMemcpy(state, tb->d_long_final, sizeof(int32_t), cudaMemcpyDeviceToHost));
    return ACB_OK;
}

extern "C" int acb_copy_records(acb_table *tb, acb_match *out, int64_t n) {
    if (!tb || n < 0 || (n && !out) || (unsigned long long)n > tb->h_out_n) { acb_set_error("bad argument"); return ACB_EINVAL; }
    if (n) memcpy(out, tb->h_out, (size_t)n * sizeof(acb_match));
    return ACB_OK;
}

/* Zero-copy hand-over of the records.  The pinned staging buffer of the last acb_scan_host can be taken by the
 * caller (no memcpy, no page faults of a fresh destination); it comes back through acb_release_records into a
 * small process-wide pool from which the next scan that needs a staging buffer is served.  A buffer that is
 * never released is simply not reused. */
namespace {
struct PinnedBuf { acb_match *p; size_t cap; };
std::mutex g_pool_mu;
std::vector<PinnedBuf> g_pool;
constexpr size_t kPoolMax = 4;

acb_match *pool_take(size_t need, size_t *cap) {
    std::lock_guard<std::mutex> lk(g_pool_mu);
    size_t best = g_pool.size();
    for (size_t i = 0; i < g_pool.size(); i++)
        if (g_pool[i].cap >= need && (best == g_pool.size() || g_pool[i].cap < g_pool[best].cap)) best = i;
    if (best == g_pool.size()) return nullptr;
    acb_match *p = g_pool[best].p;
    *cap = g_pool[best].cap;
    g_pool.erase(g_pool.begin() + (long)best);
    return p;
}
} // namespace

extern "C" int acb_take_records(acb_table *tb, acb_match **ptr, int64_t *n, int64_t *cap) {
    if (!tb || !ptr || !n || !cap) { acb_set_error("bad argument"); return ACB_EINVAL; }
    *ptr = nullptr; *n = 0; *cap = 0;
    if (tb->h_out_n == 0 || !tb->h_out) return ACB_OK;       /* nothing to hand over */
    *ptr = tb->h_out;
    *n = (int64_t)tb->h_out_n;
    *cap = (int64_t)tb->h_out_cap;
    tb->h_out = nullptr;                                     /* the next scan gets a buffer from the pool or a new one */
    tb->h_out_cap = 0;
    tb->h_out_n = 0;
    return ACB_OK;
}

extern "C" void acb_release_records(acb_match *ptr, int64_t cap) {
    if (!ptr || cap <= 0) return;
    {
        std::lock_guard<std::mutex> lk(g_pool_mu);
        if (g_pool.size() < kPoolMax) { g_pool.push_back({ptr, (size_t)cap}); return; }
    }
    cudaFreeHost(ptr);
}

/* ------------------------------------------------------------ scratch */
/* A call on stream s takes a Scratch (scratch_take): s waits for the work the last call issued on it, from any CUDA
 * stream, and a buffer too small is freed only after s has drained.  The call carves its parts from the buffer and marks
 * its own last reader (scratch_done).  scratch_wait / scratch_done also serve event-only guards (k_done). */
static int scratch_wait(cudaEvent_t done, cudaStream_t s) {
    if (done) CUDA_TRY(cudaStreamWaitEvent(s, done, 0));
    return ACB_OK;
}
static int scratch_done(cudaEvent_t *done, cudaStream_t s) {
    if (!*done) CUDA_TRY(cudaEventCreateWithFlags(done, cudaEventDisableTiming));
    CUDA_TRY(cudaEventRecord(*done, s));
    return ACB_OK;
}
static int scratch_take(Scratch &sc, size_t need, cudaStream_t s) {
    int rc = scratch_wait(sc.done, s);
    if (rc || sc.cap >= need) return rc;
    if (sc.buf) { CUDA_TRY(cudaStreamSynchronize(s)); cudaFree(sc.buf); sc.buf = nullptr; sc.cap = 0; }
    CUDA_TRY(cudaMalloc(&sc.buf, need + need / 4));
    sc.cap = need + need / 4;
    return ACB_OK;
}
/* n T's from p, 256-byte aligned (a layout of k parts needs k * 256 bytes beyond their sizes) */
template <typename T>
static T *carve(char *&p, size_t n) {
    T *r = reinterpret_cast<T *>(p);
    p += (n * sizeof(T) + 255) & ~(size_t)255;
    return r;
}

/* ------------------------------------------------------------ record sort */
/* Reference order (SURVEY 3.3): haystack, then end_index ascending, then longest key first; start order: haystack, then
 * start letter, then longest first.  One 64-bit radix key per record, hay_id | position | (max_len - len), packed into
 * the fewest bits.  When those need more than 64 bits, two stable passes: position | (max_len - len) first (kKeyEndLow,
 * kKeyStartLow), then hay_id (kKeyHay).  The leftmost-first order puts key_id where max_len - len goes: hay | start |
 * key_id (kKeyFirst), or start | key_id (kKeyFirstLow) then hay_id. */
namespace {
enum { kKeyEnd, kKeyStart, kKeyStartLow, kKeyHay, kKeyEndLow, kKeyFirst, kKeyFirstLow };

template <int kMode>
__global__ void acb_sortkey_kernel(const acb_match *rec, long long n, const int32_t *key_len, int be, int bl,
                                   int max_len, unsigned long long *keys) {
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const acb_match m = rec[i];
    if (kMode == kKeyHay) { keys[i] = (uint32_t)m.hay_id; return; }
    const int len = __ldg(key_len + m.key_id);
    const bool by_id = kMode == kKeyFirst || kMode == kKeyFirstLow;
    const unsigned long long inv = by_id ? (unsigned long long)(uint32_t)m.key_id : (unsigned long long)(max_len - len);
    const bool by_end = kMode == kKeyEnd || kMode == kKeyEndLow;
    const uint32_t pos = by_end ? (uint32_t)m.end_index : (uint32_t)(m.end_index - len + 1);
    const bool low = kMode == kKeyStartLow || kMode == kKeyEndLow || kMode == kKeyFirstLow;
    const unsigned long long hay = low ? 0ULL : (unsigned long long)(uint32_t)m.hay_id << (be + bl);
    keys[i] = hay | ((unsigned long long)pos << bl) | inv;
}
} // namespace

/* the sort key's fields: bits of the haystack, of the position and of the tie-break: max_len - key length, or (the
 * leftmost-first order) the key id, over every id of the table, removed ones included */
struct SortKey {
    int bh, be, bl, max_len;
    int bits() const { return bh + be + bl; }
};
static SortKey sort_key(const acb_table *tb, int64_t n_hay, int64_t max_hay_letters, int kind = ACB_SELECT_LONGEST) {
    auto bits_for = [](unsigned long long v) { int b = 1; while (b < 64 && (v >> b)) b++; return b; };
    const int max_len = tb->max_key_bytes / tb->L;
    const unsigned long long tie = kind == ACB_SELECT_FIRST ? (unsigned long long)std::max(tb->n_keys - 1, 0) : (unsigned long long)max_len;
    return {bits_for((unsigned long long)std::max<int64_t>(n_hay - 1, 1)), bits_for((unsigned long long)std::max<int64_t>(max_hay_letters, 1)),
            bits_for(tie), max_len};
}

/* The n records of `in` into `out`, in the order of sort-key modes kOne (one pass) / kLow (the first of two passes,
 * then hay_id).  Keys in k0 and k1 (n each); tmp: cub scratch of temp bytes, enough for a 64-bit sort of n.  Two passes
 * go through `mid`, and `out` may then be `in`. */
template <int kOne, int kLow>
static int sort_records(acb_table *tb, const SortKey &k, const acb_match *in, acb_match *mid, acb_match *out, long long n,
                        unsigned long long *k0, unsigned long long *k1, void *tmp, size_t temp, cudaStream_t s, const char *what) {
    const unsigned grid = (unsigned)((n + 255) / 256);
    const int ni = (int)n;
    size_t t = temp;
    int rc;
    if (k.bits() <= 64) {
        acb_sortkey_kernel<kOne><<<grid, 256, 0, s>>>(in, n, tb->d_keylen, k.be, k.bl, k.max_len, k0);
        if ((rc = launched(what))) return rc;
        CUDA_TRY(cub::DeviceRadixSort::SortPairs(tmp, t, k0, k1, in, out, ni, 0, k.bits(), s));
        return ACB_OK;
    }
    acb_sortkey_kernel<kLow><<<grid, 256, 0, s>>>(in, n, tb->d_keylen, k.be, k.bl, k.max_len, k0);
    if ((rc = launched(what))) return rc;
    CUDA_TRY(cub::DeviceRadixSort::SortPairs(tmp, t, k0, k1, in, mid, ni, 0, k.be + k.bl, s));
    acb_sortkey_kernel<kKeyHay><<<grid, 256, 0, s>>>(mid, n, tb->d_keylen, k.be, k.bl, k.max_len, k0);
    if ((rc = launched(what))) return rc;
    t = temp;
    CUDA_TRY(cub::DeviceRadixSort::SortPairs(tmp, t, k0, k1, mid, out, ni, 0, k.bh, s));
    return ACB_OK;
}

/* bytes of acb_sort_matches_device's scratch for n records and keys of `bits` bits; *temp: cub's part */
static size_t sort_scratch_bytes(int64_t n, int bits, cudaStream_t s, size_t *temp) {
    *temp = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, *temp, (const unsigned long long *)nullptr, (unsigned long long *)nullptr,
                                    (const acb_match *)nullptr, (acb_match *)nullptr, (int)n, 0, bits, s);
    return 4 * 256 + (size_t)n * (2 * sizeof(unsigned long long) + sizeof(acb_match)) + *temp;
}

extern "C" int acb_sort_matches_device(acb_table *tb, acb_match *d_records, int64_t n, int64_t n_hay,
                                       int64_t max_hay_letters, void *stream) {
    DeviceRestore keep_device;
    if (!tb || n < 0 || (n && !d_records)) { acb_set_error("bad argument"); return ACB_EINVAL; }
    if (n <= 1) return ACB_OK;
    /* before any allocation: scratch for this many records may not exist, and the caller sorts on the host on ERANGE */
    if (n > 0x7fffffffLL) { acb_set_error("too many records to sort on the device"); return ACB_ERANGE; }
    CUDA_TRY(cudaSetDevice(tb->device));
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    const SortKey k = sort_key(tb, n_hay, max_hay_letters);
    if (k.bits() > 64) { acb_set_error("sort key does not fit 64 bits (%d+%d+%d)", k.bh, k.be, k.bl); return ACB_ERANGE; }
    size_t temp = 0;
    int rc = scratch_take(tb->sort_buf, sort_scratch_bytes(n, k.bits(), s, &temp), s);
    if (rc != ACB_OK) return rc;
    char *p = static_cast<char *>(tb->sort_buf.buf);
    unsigned long long *k0 = carve<unsigned long long>(p, n), *k1 = carve<unsigned long long>(p, n);
    acb_match *r1 = carve<acb_match>(p, n);
    void *tmp = carve<char>(p, temp);
    if ((rc = sort_records<kKeyEnd, kKeyEndLow>(tb, k, d_records, nullptr, r1, n, k0, k1, tmp, temp, s, "sort key"))) return rc;
    CUDA_TRY(cudaMemcpyAsync(d_records, r1, (size_t)n * sizeof(acb_match), cudaMemcpyDeviceToDevice, s));
    return scratch_done(&tb->sort_buf.done, s);
}

/* ------------------------------------------------------- host-buffer scan */

template <typename T>
static int ensure(T **buf, size_t *cap, size_t need) {
    if (*cap >= need && *buf) return ACB_OK;
    if (*buf) { cudaFree(*buf); *buf = nullptr; *cap = 0; }
    size_t n = std::max<size_t>(need + need / 4, 1024);
    CUDA_TRY(cudaMalloc(reinterpret_cast<void **>(buf), n * sizeof(T)));
    *cap = n;
    return ACB_OK;
}

/* pinned staging for n records (from the pool some caller has given back, or new) */
static int ensure_pinned_out(acb_table *tb, size_t n) {
    if (tb->h_out_cap >= n && tb->h_out) return ACB_OK;
    if (tb->h_out) { acb_release_records(tb->h_out, (int64_t)tb->h_out_cap); tb->h_out = nullptr; tb->h_out_cap = 0; }
    size_t got = 0;
    if (acb_match *p = pool_take(n, &got)) {
        tb->h_out = p;
        tb->h_out_cap = got;
    } else {
        size_t want = n + n / 4 + 1024;
        CUDA_TRY(cudaMallocHost(reinterpret_cast<void **>(&tb->h_out), want * sizeof(acb_match)));
        tb->h_out_cap = want;
    }
    return ACB_OK;
}

/* host offsets of n haystacks: non-decreasing multiples of the letter width, from 0 to total.  The kernels read
 * hay[offsets[i] .. offsets[i+1]) unchecked. */
static int check_offsets(int32_t L, const int64_t *offsets, int64_t n, int64_t total) {
    bool ok = offsets[0] == 0 && offsets[n] == total;
    for (int64_t i = 0; ok && i < n; i++) ok = offsets[i + 1] >= offsets[i] && offsets[i + 1] % L == 0;
    if (ok) return ACB_OK;
    acb_set_error("offsets must be non-decreasing multiples of letter_bytes, start at 0 and end at the total byte count");
    return ACB_EINVAL;
}

/* The host routes' workspace on tb->stream: the device set, the stream and the count words made, tb->w_hay grown for
 * total bytes and tb->w_off for the offsets of n haystacks when there are offsets. */
static int host_workspace(acb_table *tb, int64_t total, const int64_t *offsets, int64_t n) {
    CUDA_TRY(cudaSetDevice(tb->device));
    if (!tb->stream) CUDA_TRY(cudaStreamCreateWithFlags(&tb->stream, cudaStreamNonBlocking));
    if (!tb->w_count) CUDA_TRY(cudaMalloc(reinterpret_cast<void **>(&tb->w_count), sizeof(unsigned long long)));
    if (!tb->h_count) CUDA_TRY(cudaMallocHost(reinterpret_cast<void **>(&tb->h_count), sizeof(unsigned long long)));
    int rc;
    if ((rc = ensure(&tb->w_hay, &tb->w_hay_cap, (size_t)total + 64))) return rc;
    if (offsets && (rc = ensure(&tb->w_off, &tb->w_off_cap, (size_t)n + 1))) return rc;
    return ACB_OK;
}

/* ... and the batch and its offsets on their way up, asynchronously; *d_off = the device offsets, or nullptr */
static int upload_batch(acb_table *tb, const uint8_t *hay, int64_t total, const int64_t *offsets, int64_t n, const int64_t **d_off) {
    int rc = host_workspace(tb, total, offsets, n);
    if (rc != ACB_OK) return rc;
    *d_off = nullptr;
    if (total) CUDA_TRY(cudaMemcpyAsync(tb->w_hay, hay, (size_t)total, cudaMemcpyHostToDevice, tb->stream));
    if (offsets) {
        CUDA_TRY(cudaMemcpyAsync(tb->w_off, offsets, (size_t)(n + 1) * sizeof(long long), cudaMemcpyHostToDevice, tb->stream));
        *d_off = reinterpret_cast<const int64_t *>(tb->w_off);
    }
    return ACB_OK;
}

/* the reference order of records (SURVEY 3.3): haystack, then end_index ascending, then longest key first (fail-chain order) */
struct RefOrder {
    const int32_t *key_len;
    bool operator()(const acb_match &a, const acb_match &b) const {
        if (a.hay_id != b.hay_id) return a.hay_id < b.hay_id;
        if (a.end_index != b.end_index) return a.end_index < b.end_index;
        if (key_len[a.key_id] != key_len[b.key_id]) return key_len[a.key_id] > key_len[b.key_id];
        return a.key_id < b.key_id;                            /* equal lengths at one end: case variants (alias expansion) */
    }
};

/* The host routes' last step, on s: the record count at d_n to the host (a wait), ACB_EOVERFLOW with the exact count
 * past cap, then the records of d_rec into the pinned staging buffer and into `out` when given.  With sort they are put
 * into the reference order first: on the device, or on the host when the device sort's key does not fit 64 bits. */
static int read_back(acb_table *tb, const unsigned long long *d_n, acb_match *d_rec, int64_t cap, int sort, int64_t n_hay,
                     int64_t max_letters, acb_match *out, int64_t *n_found, cudaStream_t s) {
    CUDA_TRY(cudaMemcpyAsync(tb->h_count, d_n, sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    const unsigned long long n = *tb->h_count;
    *n_found = (int64_t)n;
    if (n > (unsigned long long)cap) {
        acb_set_error("match buffer too small: %llu matches, capacity %lld", n, (long long)cap);
        return ACB_EOVERFLOW;
    }
    if (n) {
        int rc;
        if ((rc = ensure_pinned_out(tb, (size_t)n))) return rc;
        bool host_sort = false;
        if (sort && (rc = acb_sort_matches_device(tb, d_rec, (int64_t)n, n_hay, max_letters, s)) != ACB_OK) {
            if (rc != ACB_ERANGE) return rc;
            host_sort = true;
        }
        CUDA_TRY(cudaMemcpyAsync(tb->h_out, d_rec, (size_t)n * sizeof(acb_match), cudaMemcpyDeviceToHost, s));
        CUDA_TRY(cudaStreamSynchronize(s));
        if (host_sort) std::sort(tb->h_out, tb->h_out + n, RefOrder{tb->key_len.data()});
        if (out) memcpy(out, tb->h_out, (size_t)n * sizeof(acb_match));   /* out == NULL: fetch with acb_copy_records */
    }
    tb->h_out_n = n;
    return ACB_OK;
}

/* The host-buffer scan as a pipeline over 32 MiB chunks of the batch: chunk c is copied to the device on the copy
 * stream while the stream kernel scans the start positions the copy of chunk c-1 completed, and its records are sorted
 * and copied back (the other PCIe direction) while later chunks are still going up.  A start position belongs to the
 * chunk in which a key of maximal length starting there ends, so a launch never needs bytes that are not on the device
 * yet.  Chunks are in position order and each is sorted by itself; only the one haystack a chunk boundary cuts can have
 * its records out of order across the cut, and those two adjacent runs are merged on the host at the end. */
static int scan_host_pipelined(acb_table *tb, const uint8_t *hay, int64_t total, const int64_t *offsets, int64_t n_hay,
                               int64_t stride_bytes, int64_t cap, int64_t *n_found, int sort) {
    constexpr long long kChunk = 32LL << 20;
    const int nch = (int)((total + kChunk - 1) / kChunk);
    if (!tb->s_copy) CUDA_TRY(cudaStreamCreateWithFlags(&tb->s_copy, cudaStreamNonBlocking));
    if (!tb->s_sort) CUDA_TRY(cudaStreamCreateWithFlags(&tb->s_sort, cudaStreamNonBlocking));
    while ((int)tb->ev_h2d.size() < nch) {
        cudaEvent_t a, b;
        CUDA_TRY(cudaEventCreateWithFlags(&a, cudaEventDisableTiming));
        CUDA_TRY(cudaEventCreateWithFlags(&b, cudaEventDisableTiming));
        tb->ev_h2d.push_back(a);
        tb->ev_scan.push_back(b);
    }
    if (tb->h_counts_cap < (size_t)nch) {
        if (tb->h_counts) cudaFreeHost(tb->h_counts);
        tb->h_counts = nullptr;
        CUDA_TRY(cudaMallocHost(reinterpret_cast<void **>(&tb->h_counts), (size_t)(nch + 16) * sizeof(unsigned long long)));
        tb->h_counts_cap = (size_t)nch + 16;
    }
    int rc;
    if ((rc = ensure_pinned_out(tb, (size_t)cap))) return rc;
    const int64_t max_letters = (offsets ? total : stride_bytes) / tb->L;
    size_t temp = 0;                                            /* scratch of the per-chunk sorts, once, before anything is in flight */
    if (sort && (rc = scratch_take(tb->sort_buf, sort_scratch_bytes(cap, 64, tb->s_sort, &temp), tb->s_sort))) return rc;
    cudaStream_t sc = tb->stream, sh = tb->s_copy, ss = tb->s_sort;
    const int64_t *d_off = nullptr;
    if (offsets) {
        CUDA_TRY(cudaMemcpyAsync(tb->w_off, offsets, (size_t)(n_hay + 1) * sizeof(long long), cudaMemcpyHostToDevice, sh));
        d_off = reinterpret_cast<const int64_t *>(tb->w_off);
    }
    for (int c = 0; c < nch; c++) {
        const long long b0 = (long long)c * kChunk, b1 = std::min<long long>(b0 + kChunk, total);
        CUDA_TRY(cudaMemcpyAsync(tb->w_hay + b0, hay + b0, (size_t)(b1 - b0), cudaMemcpyHostToDevice, sh));
        CUDA_TRY(cudaEventRecord(tb->ev_h2d[c], sh));
    }
    CUDA_TRY(cudaMemsetAsync(tb->w_count, 0, sizeof(unsigned long long), sc));
    ScanParams p;
    fill_params(tb, p, tb->w_hay, total, d_off, n_hay, stride_bytes, tb->w_out, cap, reinterpret_cast<int64_t *>(tb->w_count));
    const long long reach = ((long long)tb->max_key_bytes + 31) & ~31LL;      /* a start position this far before a cut waits for the next chunk */
    auto cut = [&](int c) { return c <= 0 ? 0LL : (c >= nch ? (long long)total : std::max<long long>(0, (long long)c * kChunk - reach)); };
    for (int c = 0; c < nch; c++) {
        CUDA_TRY(cudaStreamWaitEvent(sc, tb->ev_h2d[c], 0));
        if (tb->fold) {                                         /* in place: only this scan reads the batch's copy */
            const long long b0 = (long long)c * kChunk, b1 = std::min<long long>(b0 + kChunk, total);
            if ((rc = fold_text(tb, tb->w_hay + b0, tb->w_hay + b0, b1 - b0, sc))) return rc;
        }
        if (cut(c + 1) > cut(c) && (rc = launch_filter_range(tb, p, cut(c), cut(c + 1), sc))) return rc;
        CUDA_TRY(cudaMemcpyAsync(tb->h_counts + c, tb->w_count, sizeof(unsigned long long), cudaMemcpyDeviceToHost, sc));
        CUDA_TRY(cudaEventRecord(tb->ev_scan[c], sc));
    }
    unsigned long long prev = 0;
    for (int c = 0; c < nch; c++) {
        CUDA_TRY(cudaEventSynchronize(tb->ev_scan[c]));
        const unsigned long long cur = std::min<unsigned long long>(tb->h_counts[c], (unsigned long long)cap);
        if (cur > prev) {
            if (sort && (rc = acb_sort_matches_device(tb, tb->w_out + prev, (int64_t)(cur - prev), n_hay, max_letters, ss))) return rc;
            CUDA_TRY(cudaMemcpyAsync(tb->h_out + prev, tb->w_out + prev, (size_t)(cur - prev) * sizeof(acb_match), cudaMemcpyDeviceToHost, ss));
        }
        prev = cur;
    }
    CUDA_TRY(cudaStreamSynchronize(ss));
    const unsigned long long n = tb->h_counts[nch - 1];
    *n_found = (int64_t)n;
    if (n > (unsigned long long)cap) {
        acb_set_error("match buffer too small: %llu matches, capacity %lld", n, (long long)cap);
        return ACB_EOVERFLOW;
    }
    if (sort) {                                                 /* the haystack every cut goes through: merge its two runs */
        for (int c = 0; c + 1 < nch; c++) {
            const unsigned long long mid = tb->h_counts[c];
            if (mid == 0 || mid >= n) continue;
            const int32_t h = tb->h_out[mid - 1].hay_id;          /* the last haystack of chunk c; the cut lies in it or right after it */
            if (tb->h_out[mid].hay_id != h) continue;
            unsigned long long lo = mid, hi = mid;
            while (lo > 0 && tb->h_out[lo - 1].hay_id == h) lo--;
            const unsigned long long stop = std::min<unsigned long long>(n, tb->h_counts[c + 1]);   /* this cut's run ends with chunk c+1; a longer haystack meets the next cut */
            while (hi < stop && tb->h_out[hi].hay_id == h) hi++;
            std::inplace_merge(tb->h_out + lo, tb->h_out + mid, tb->h_out + hi, RefOrder{tb->key_len.data()});
        }
    }
    tb->h_out_n = n;
    return ACB_OK;
}

struct WordSet;
static int scan_host_full(acb_table *tb, const uint8_t *hay, int64_t total_bytes, const int64_t *offsets, int64_t n_hay,
                          int64_t stride_bytes, const WordSet *ws, acb_match *out, int64_t cap, int64_t *n_found, int algo, int sort);

extern "C" int acb_scan_host(acb_table *tb, const uint8_t *hay, int64_t total_bytes,
                             const int64_t *offsets, int64_t n_hay, int64_t stride_bytes,
                             acb_match *out, int64_t cap, int64_t *n_found, int algo, int sort) {
    DeviceRestore keep_device;
    if (!tb || !n_found || total_bytes < 0 || n_hay < 0 || cap < 0) { acb_set_error("bad argument"); return ACB_EINVAL; }
    if (algo == ACB_ALGO_LONG && refuse_folded(tb, "ACB_ALGO_LONG")) return ACB_EINVAL;
    if (tb->n_alias)                                             /* the full list, expanded; not pipelined */
        return scan_host_full(tb, hay, total_bytes, offsets, n_hay, stride_bytes, nullptr, out, cap, n_found, algo, sort);
    *n_found = 0;
    tb->h_out_n = 0;
    if (total_bytes == 0 || n_hay == 0) {
        if (algo == ACB_ALGO_LONG) long_scan_without_launch(tb);
        return ACB_OK;
    }
    int rc;
    if ((rc = host_workspace(tb, total_bytes, offsets, n_hay)) || (rc = ensure(&tb->w_out, &tb->w_out_cap, (size_t)std::max<int64_t>(cap, 1))))
        return rc;
    const int64_t max_letters = (offsets ? total_bytes : stride_bytes) / tb->L;
    {   /* large batches on the fast path: copy, scan, sort and copy-back as a pipeline over chunks */
        const int bits = sort_key(tb, n_hay, max_letters).bits();
        static const bool no_pipe = getenv("ACB_NO_PIPELINE") != nullptr;
        if (!no_pipe && (algo == ACB_ALGO_AUTO || algo == ACB_ALGO_FILTER) && tb->n_keys > 0 && total_bytes >= (48LL << 20) && bits <= 64 && cap < 0x7fffffffLL) {
            rc = scan_host_pipelined(tb, hay, total_bytes, offsets, n_hay, stride_bytes, cap, n_found, sort);
            if (rc == ACB_OK && out && *n_found) memcpy(out, tb->h_out, (size_t)*n_found * sizeof(acb_match));
            return rc;
        }
    }
    static const bool trace = getenv("ACB_TRACE") != nullptr;          /* phase timing to stderr (adds syncs) */
    auto now = [] { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
    double t0 = trace ? now() : 0, t1 = 0, t2 = 0;
    const int64_t *d_off = nullptr;
    if ((rc = upload_batch(tb, hay, total_bytes, offsets, n_hay, &d_off))) return rc;
    cudaStream_t s = tb->stream;
    CUDA_TRY(cudaMemsetAsync(tb->w_count, 0, sizeof(unsigned long long), s));
    if (trace) { cudaStreamSynchronize(s); t1 = now(); }
    rc = acb_scan_device(tb, tb->w_hay, total_bytes, d_off, n_hay, stride_bytes, tb->w_out, cap, reinterpret_cast<int64_t *>(tb->w_count), s, algo);
    if (rc != ACB_OK) return rc;
    if (trace) { cudaStreamSynchronize(s); t2 = now(); }
    rc = read_back(tb, tb->w_count, tb->w_out, cap, sort, n_hay, max_letters, out, n_found, s);
    if (trace && rc == ACB_OK)
        fprintf(stderr, "[acb_scan_host] %lld B: h2d %.3f ms, scan %.3f ms, sort+d2h+copy %.3f ms (%lld records)\n",
                (long long)total_bytes, t1 - t0, t2 - t1, now() - t2, (long long)*n_found);
    return rc;
}

/* ------------------------------------------------------------ white space */
/* iter(..., ignore_white_space=1) for a batch: compact, scan, map back.  acb_compact_kernel drops the letters of the
 * skip set from the flat buffer in one pass (tile ids from a counter, decoupled look-back over per-tile kept counts,
 * kept letters staged in shared memory so the stores are coalesced) and leaves what the map back needs: one keep mask
 * per 32-letter group, a uint16 prefix per group within its tile and an int64 prefix per tile -- 6 bytes per 32 letters
 * plus 16 per tile, never the text again.  The ordinary scan kernels then run on the compacted haystacks unchanged;
 * acb_remap_kernel turns a record's compacted letter into the original one with a binary search over tiles, one over
 * the tile's groups and __fns on one mask. */
namespace {
constexpr int kCmpThreads = 256;                          /* one 32-letter group per thread */
constexpr int kCmpTile = kCmpThreads * 32;                /* letters per tile (uint16 prefixes within a tile) */
constexpr unsigned long long kLbAgg = 1ULL << 62, kLbPre = 2ULL << 62, kLbVal = (1ULL << 62) - 1;

struct CompactMeta {
    const uint32_t *mask;
    const uint16_t *gpre;
    const long long *tile_pre;    /* [n_tiles + 1] */
    long long n_tiles;
};

struct CompactParams {
    const uint8_t *in;
    uint8_t *out;                 /* 16-byte aligned */
    long long n_letters;
    uint32_t *mask;
    uint16_t *gpre;
    long long *tile_pre;
    unsigned long long *status;   /* [n_tiles], zeroed */
    unsigned int *ctr;            /* zeroed */
    long long n_tiles;
    const uint32_t *set;          /* L > 1: the sorted skip set */
    int n_set;
    uint32_t bits[8];             /* L == 1: the skip set as a 256-bit table */
};

template <typename T>
__device__ __forceinline__ bool skip_letter(T v, const uint32_t *bits, const uint32_t *set, int n) {
    if (sizeof(T) == 1) return (bits[v >> 5] >> (v & 31)) & 1;
    int lo = 0, hi = n;                                    /* the set is short: a binary search in shared memory */
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (set[mid] < (uint32_t)v) lo = mid + 1; else hi = mid;
    }
    return lo < n && set[lo] == (uint32_t)v;
}

template <typename T>
__global__ void __launch_bounds__(kCmpThreads, 4) acb_compact_kernel(const __grid_constant__ CompactParams p) {
    using Scan = cub::BlockScan<int, kCmpThreads>;
    __shared__ typename Scan::TempStorage scan_tmp;
    __shared__ __align__(16) uint8_t s_buf[kCmpTile * sizeof(T) + 16];   /* the tile's kept letters */
    __shared__ uint32_t s_set[sizeof(T) == 1 ? 1 : ACB_MAX_SKIP];
    __shared__ uint32_t s_bits[8];
    __shared__ long long s_tile, s_base;
    if (threadIdx.x == 0) s_tile = atomicAdd(p.ctr, 1u);   /* in claim order: every earlier tile is running or done */
    if (sizeof(T) == 1) { if (threadIdx.x < 8) s_bits[threadIdx.x] = p.bits[threadIdx.x]; }
    else for (int i = threadIdx.x; i < p.n_set; i += kCmpThreads) s_set[i] = __ldg(p.set + i);
    __syncthreads();
    const long long tile = s_tile, t0 = tile * kCmpTile;
    const int n_tile = (int)min((long long)kCmpTile, p.n_letters - t0);
    constexpr int kWords = 8 * (int)sizeof(T), kPer = 4 / (int)sizeof(T);
    uint32_t w[kWords];                                    /* this thread's 32 letters, straight into registers */
    const long long first = t0 + (long long)threadIdx.x * 32;
    if (first + 32 <= p.n_letters) {                       /* 32 * sizeof(T) bytes at a 32-byte aligned offset, read once */
        const uint4 *src = reinterpret_cast<const uint4 *>(p.in + first * (long long)sizeof(T));
#pragma unroll
        for (int k = 0; k < kWords / 4; k++) {
            const uint4 v = __ldcs(src + k);
            w[4 * k] = v.x; w[4 * k + 1] = v.y; w[4 * k + 2] = v.z; w[4 * k + 3] = v.w;
        }
    } else {
        const T *src = reinterpret_cast<const T *>(p.in);
#pragma unroll
        for (int k = 0; k < kWords; k++) w[k] = 0;
#pragma unroll
        for (int j = 0; j < 32; j++)
            if (first + j < p.n_letters) w[j / kPer] |= (uint32_t)src[first + j] << (8 * (int)sizeof(T) * (j % kPer));
    }
    const int valid = n_tile - (int)threadIdx.x * 32;      /* letters of this group inside the batch */
    uint32_t keep = 0;
#pragma unroll
    for (int j = 0; j < 32; j++) {
        const T v = (T)(w[j / kPer] >> (8 * (int)sizeof(T) * (j % kPer)));
        if (j < valid && !skip_letter<T>(v, s_bits, s_set, p.n_set)) keep |= 1u << j;
    }
    int pre, agg;
    Scan(scan_tmp).ExclusiveSum(__popc(keep), pre, agg);
    const long long g = tile * kCmpThreads + threadIdx.x;
    p.mask[g] = keep;
    p.gpre[g] = (uint16_t)pre;
    T *kept = reinterpret_cast<T *>(s_buf);
    int o = pre;
#pragma unroll
    for (int j = 0; j < 32; j++)
        if ((keep >> j) & 1) kept[o++] = (T)(w[j / kPer] >> (8 * (int)sizeof(T) * (j % kPer)));
    if (threadIdx.x == 0) {                                /* decoupled look-back over the tiles before this one */
        long long base = 0;
        if (tile == 0) {
            atomicExch(p.status, kLbPre | (unsigned long long)agg);
        } else {
            atomicExch(p.status + tile, kLbAgg | (unsigned long long)agg);
            for (long long i = tile - 1;; --i) {
                unsigned long long st;
                while ((st = *reinterpret_cast<volatile unsigned long long *>(p.status + i)) == 0) {}
                base += (long long)(st & kLbVal);
                if (st & kLbPre) break;
            }
            atomicExch(p.status + tile, kLbPre | (unsigned long long)(base + agg));
        }
        p.tile_pre[tile] = base;
        if (tile == p.n_tiles - 1) p.tile_pre[p.n_tiles] = base + agg;
        s_base = base;
    }
    __syncthreads();
    /* coalesced stores: bytes up to a 16-byte boundary of the destination, then 16-byte words, then the rest */
    uint8_t *dst = p.out + s_base * (long long)sizeof(T);
    const int nb = agg * (int)sizeof(T);
    const int head = min(nb, (int)((16 - (reinterpret_cast<uintptr_t>(dst) & 15)) & 15)), nmid = (nb - head) >> 4;
    if ((int)threadIdx.x < head) dst[threadIdx.x] = s_buf[threadIdx.x];
    const int sh = (head & 3) * 8;
    const uint32_t *sw = reinterpret_cast<const uint32_t *>(s_buf) + (head >> 2);
    for (int i = threadIdx.x; i < nmid; i += kCmpThreads) {
        const uint32_t *q = sw + 4 * i;                    /* unaligned by head bytes in shared memory: funnel shifts */
        const uint32_t a0 = q[0], a1 = q[1], a2 = q[2], a3 = q[3], a4 = q[4];
        reinterpret_cast<uint4 *>(dst + head)[i] = make_uint4(__funnelshift_r(a0, a1, sh), __funnelshift_r(a1, a2, sh),
                                                              __funnelshift_r(a2, a3, sh), __funnelshift_r(a3, a4, sh));
    }
    for (int i = head + (nmid << 4) + threadIdx.x; i < nb; i += kCmpThreads) dst[i] = s_buf[i];
}

/* kept letters before letter q of the original buffer */
__device__ __forceinline__ long long kept_before(const CompactMeta &m, long long q) {
    const long long t = q / kCmpTile;
    if (t >= m.n_tiles) return __ldg(m.tile_pre + m.n_tiles);
    const long long g = q >> 5;
    return __ldg(m.tile_pre + t) + __ldg(m.gpre + g) + __popc(__ldg(m.mask + g) & ((1u << (q & 31)) - 1u));
}

/* coff[h] = compacted byte offset of haystack h, h = 0 .. n_hay */
__global__ void acb_compact_offsets_kernel(const CompactMeta m, const long long *off, long long stride, long long n_hay, int ls,
                                           long long *coff) {
    const long long h = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (h > n_hay) return;
    coff[h] = kept_before(m, hay_start(off, stride, h) >> ls) << ls;
}

/* the stored records (min(*count, cap)) from compacted letters of their haystack to original ones */
__global__ void acb_remap_kernel(const CompactMeta m, const long long *coff, const long long *off, long long stride, int ls,
                                 acb_match *rec, const unsigned long long *count, long long cap) {
    const long long n = (long long)min(*count, (unsigned long long)cap);
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        acb_match r = rec[i];
        const long long k = (__ldg(coff + r.hay_id) >> ls) + r.end_index;     /* rank of the kept letter */
        long long lo = 0, hi = m.n_tiles;                  /* the last tile with tile_pre <= k holds it */
        while (hi - lo > 1) { const long long mid = (lo + hi) >> 1; if (__ldg(m.tile_pre + mid) <= k) lo = mid; else hi = mid; }
        const long long kt = k - __ldg(m.tile_pre + lo);
        int a = 0, b = kCmpThreads;                        /* ... and its last group with gpre <= kt */
        const uint16_t *gp = m.gpre + lo * kCmpThreads;
        while (b - a > 1) { const int mid = (a + b) >> 1; if ((long long)__ldg(gp + mid) <= kt) a = mid; else b = mid; }
        const long long g = lo * kCmpThreads + a;
        const int bit = (int)__fns(__ldg(m.mask + g), 0, (int)(kt - __ldg(gp + a)) + 1);
        r.end_index = (int32_t)(g * 32 + bit - (hay_start(off, stride, r.hay_id) >> ls));
        rec[i] = r;
    }
}
} // namespace

extern "C" int acb_last_skip_ms(float *compact_ms, float *remap_ms) {
    if (!compact_ms || !remap_ms) { acb_set_error("bad argument"); return ACB_EINVAL; }
    *compact_ms = g_compact_ms;
    *remap_ms = g_remap_ms;
    return ACB_OK;
}

static int check_skip(const uint32_t *skip, int64_t n_skip, int algo) {
    if (algo == ACB_ALGO_LONG) { acb_set_error("iter_long has no white-space skipping"); return ACB_EINVAL; }
    if (n_skip < 0 || n_skip > ACB_MAX_SKIP || (n_skip && !skip)) { acb_set_error("skip set of %lld letters (at most %d)", (long long)n_skip, ACB_MAX_SKIP); return ACB_EINVAL; }
    for (int64_t i = 1; i < n_skip; i++)
        if (skip[i] <= skip[i - 1]) { acb_set_error("skip set not sorted and distinct at %lld", (long long)i); return ACB_EINVAL; }
    return ACB_OK;
}

/* Compact total_bytes of d_in (16-byte aligned) into tb->k_buf and the haystack offsets into tb->k_coff; *kept_bytes
 * is the compacted size (this waits for the compaction on s).  The map-back metadata stays in tb->k_*. */
static int compact(acb_table *tb, const uint8_t *d_in, int64_t total, const int64_t *d_off, int64_t n_hay, int64_t stride,
                   const uint32_t *skip, int64_t n_skip, cudaStream_t s, long long *kept_bytes, CompactMeta *meta) {
    const int L = tb->L, ls = L == 4 ? 2 : (L == 2 ? 1 : 0);
    const long long n_letters = total / L, n_tiles = (n_letters + kCmpTile - 1) / kCmpTile;
    int rc;
    if ((rc = ensure(&tb->k_buf, &tb->k_buf_cap, (size_t)total + 64)) || (rc = ensure(&tb->k_mask, &tb->k_mask_cap, (size_t)n_tiles * kCmpThreads)) ||
        (rc = ensure(&tb->k_gpre, &tb->k_gpre_cap, (size_t)n_tiles * kCmpThreads)) || (rc = ensure(&tb->k_tile_pre, &tb->k_tile_pre_cap, (size_t)n_tiles + 1)) ||
        (rc = ensure(&tb->k_status, &tb->k_status_cap, (size_t)n_tiles)) || (rc = ensure(&tb->k_coff, &tb->k_coff_cap, (size_t)n_hay + 1)))
        return rc;
    if (!tb->k_set) CUDA_TRY(cudaMalloc(reinterpret_cast<void **>(&tb->k_set), ACB_MAX_SKIP * sizeof(uint32_t)));
    if (!tb->k_ctr) CUDA_TRY(cudaMalloc(reinterpret_cast<void **>(&tb->k_ctr), sizeof(unsigned int)));
    if (!tb->h_kept) CUDA_TRY(cudaMallocHost(reinterpret_cast<void **>(&tb->h_kept), sizeof(long long)));
    if ((rc = scratch_wait(tb->k_done, s))) return rc;
    g_compact_ms = g_remap_ms = 0.f;
    CompactParams p;
    memset(&p, 0, sizeof(p));
    p.in = d_in; p.out = tb->k_buf; p.n_letters = n_letters;
    p.mask = tb->k_mask; p.gpre = tb->k_gpre; p.tile_pre = tb->k_tile_pre; p.status = tb->k_status; p.ctr = tb->k_ctr;
    p.n_tiles = n_tiles; p.set = tb->k_set; p.n_set = (int)n_skip;
    for (int64_t i = 0; i < n_skip; i++) if (skip[i] < 256) p.bits[skip[i] >> 5] |= 1u << (skip[i] & 31);
    if (L > 1 && n_skip) CUDA_TRY(cudaMemcpyAsync(tb->k_set, skip, (size_t)n_skip * sizeof(uint32_t), cudaMemcpyHostToDevice, s));
    CUDA_TRY(cudaMemsetAsync(tb->k_status, 0, (size_t)n_tiles * sizeof(unsigned long long), s));
    CUDA_TRY(cudaMemsetAsync(tb->k_ctr, 0, sizeof(unsigned int), s));
    if (n_tiles > 0x7fffffffLL) { acb_set_error("batch too large to compact in one launch"); return ACB_ERANGE; }
    if ((rc = timing_mark(&tb->k_t0, s))) return rc;
    with_width(L, [&](auto w) {
        using T = std::conditional_t<w.value == 1, uint8_t, std::conditional_t<w.value == 2, uint16_t, uint32_t>>;
        acb_compact_kernel<T><<<(unsigned)n_tiles, kCmpThreads, 0, s>>>(p);
    });
    CUDA_TRY(cudaGetLastError());
    if ((rc = timing_mark(&tb->k_t1, s)) || (rc = timing_ms(tb->k_t0, tb->k_t1, &g_compact_ms))) return rc;
    meta->mask = tb->k_mask; meta->gpre = tb->k_gpre; meta->tile_pre = tb->k_tile_pre; meta->n_tiles = n_tiles;
    acb_compact_offsets_kernel<<<(unsigned)((n_hay + 1 + 255) / 256), 256, 0, s>>>(*meta, reinterpret_cast<const long long *>(d_off), stride,
                                                                                 n_hay, ls, tb->k_coff);
    if ((rc = launched("compaction offsets", 2))) return rc;
    CUDA_TRY(cudaMemcpyAsync(tb->h_kept, tb->k_tile_pre + n_tiles, sizeof(long long), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    *kept_bytes = *tb->h_kept * L;
    return ACB_OK;
}

static int launch_remap(acb_table *tb, const CompactMeta &meta, const int64_t *d_off, int64_t stride, acb_match *d_out, int64_t cap,
                        int64_t *d_count, cudaStream_t s) {
    if (cap <= 0) return ACB_OK;
    const int ls = tb->L == 4 ? 2 : (tb->L == 2 ? 1 : 0);
    int rc;
    if ((rc = timing_mark(&tb->k_t0, s))) return rc;
    acb_remap_kernel<<<blocks(tb, cap), 256, 0, s>>>(meta, tb->k_coff, reinterpret_cast<const long long *>(d_off), stride, ls, d_out,
                                                    reinterpret_cast<const unsigned long long *>(d_count), cap);
    if ((rc = launched("remap kernel")) || (rc = timing_mark(&tb->k_t1, s))) return rc;
    return timing_ms(tb->k_t0, tb->k_t1, &g_remap_ms);
}

extern "C" int acb_scan_device_skip(acb_table *tb, const uint8_t *d_hay, int64_t total_bytes,
                                    const int64_t *d_offsets, int64_t n_hay, int64_t stride_bytes,
                                    acb_match *d_out, int64_t cap, int64_t *d_count, void *stream, int algo,
                                    const uint32_t *skip, int64_t n_skip) {
    DeviceRestore keep_device;
    if (!tb || !d_count || total_bytes < 0 || n_hay < 0 || cap < 0 || (cap > 0 && !d_out)) { acb_set_error("bad argument"); return ACB_EINVAL; }
    if (refuse_folded(tb, "a white-space scan")) return ACB_EINVAL;
    int rc = check_skip(skip, n_skip, algo);
    if (rc != ACB_OK) return rc;
    if (n_hay > 0x7fffffffLL) { acb_set_error("more than 2^31-1 haystacks in one batch"); return ACB_ERANGE; }
    if (!d_offsets && (rc = check_stride(tb->L, total_bytes, n_hay, stride_bytes, 1))) return rc;
    CUDA_TRY(cudaSetDevice(tb->device));
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    CUDA_TRY(cudaMemsetAsync(d_count, 0, sizeof(int64_t), s));
    if (n_skip == 0) return acb_scan_device(tb, d_hay, total_bytes, d_offsets, n_hay, stride_bytes, d_out, cap, d_count, stream, algo);
    if (total_bytes == 0 || n_hay == 0 || tb->n_keys == 0) return ACB_OK;
    if (reinterpret_cast<uintptr_t>(d_hay) & 15) { acb_set_error("d_hay must be 16-byte aligned"); return ACB_EINVAL; }
    long long kept = 0;
    CompactMeta meta;
    if ((rc = compact(tb, d_hay, total_bytes, d_offsets, n_hay, stride_bytes, skip, n_skip, s, &kept, &meta))) return rc;
    if (kept == 0) return ACB_OK;
    if ((rc = acb_scan_device(tb, tb->k_buf, kept, reinterpret_cast<const int64_t *>(tb->k_coff), n_hay, 0, d_out, cap, d_count, stream, algo))) return rc;
    if ((rc = launch_remap(tb, meta, d_offsets, stride_bytes, d_out, cap, d_count, s))) return rc;
    return scratch_done(&tb->k_done, s);                   /* the remap was the last reader of the k_* workspace */
}

extern "C" int acb_scan_host_skip(acb_table *tb, const uint8_t *hay, int64_t total_bytes,
                                  const int64_t *offsets, int64_t n_hay, int64_t stride_bytes,
                                  acb_match *out, int64_t cap, int64_t *n_found, int algo, int sort,
                                  const uint32_t *skip, int64_t n_skip) {
    DeviceRestore keep_device;
    if (!tb || !n_found || total_bytes < 0 || n_hay < 0 || cap < 0 || (total_bytes && !hay)) { acb_set_error("bad argument"); return ACB_EINVAL; }
    if (refuse_folded(tb, "a white-space scan")) return ACB_EINVAL;
    *n_found = 0;
    int rc = check_skip(skip, n_skip, algo);
    if (rc != ACB_OK) return rc;
    tb->h_out_n = 0;
    if (total_bytes == 0 || n_hay == 0) return ACB_OK;
    const int64_t *d_off = nullptr;
    if ((rc = upload_batch(tb, hay, total_bytes, offsets, n_hay, &d_off)) || (rc = ensure(&tb->w_out, &tb->w_out_cap, (size_t)std::max<int64_t>(cap, 1))))
        return rc;
    cudaStream_t s = tb->stream;
    if ((rc = acb_scan_device_skip(tb, tb->w_hay, total_bytes, d_off, n_hay, stride_bytes, tb->w_out, cap, reinterpret_cast<int64_t *>(tb->w_count), s,
                                   algo, skip, n_skip)))
        return rc;
    return read_back(tb, tb->w_count, tb->w_out, cap, sort, n_hay, (offsets ? total_bytes : stride_bytes) / tb->L, out, n_found, s);
}

/* ------------------------------------------------------------ stream batches */
/* A stream batch (acb_streams) keeps every stream's carry-over in HBM: the number of letters consumed, and either the
 * last T = longest_word - 1 letters (find_all semantics) or the walk state (iter_long semantics).  A feed scans the
 * chunks themselves with the ordinary scan (acb_scan_device: every match that starts and ends inside a chunk), then one
 * lane per chunk walks the goto/fail automaton over the chunk's seam -- its stream's tail followed by the first
 * min(T, n) letters of the chunk -- and reports only the matches that start in the tail and end in the chunk.  A match
 * that ends in the chunk but starts before it has at most T + 1 letters, so at most T of them lie in the chunk and the
 * seam holds all of it; a chunk shorter than T is covered by the next feed, whose tail is the last T letters of
 * tail || chunk.  The new tails (long mode: end states) go to per-feed staging; a commit kernel copies them into the
 * streams and advances the positions only when the feed's records fit the caller's buffer, so a feed that overflows
 * changes no stream and can be repeated with a larger buffer. */
namespace {
struct StreamsArgs {
    const int32_t *ids;           /* chunk -> stream; nullptr: chunk h continues stream h */
    long long n_streams;
    long long *pos;               /* [n_streams] letters consumed since the start / the last reset */
    long long *kept;              /* with a skip set: [n_streams] letters consumed that were kept (the tail counts those);
                                     nullptr: every letter is kept, pos serves */
    uint8_t *tail;                /* [n_streams][T letters]: the last min(T, pos) letters consumed, left aligned */
    uint8_t *next_tail;           /* [n_chunks][T letters]: the tail after this feed's chunk (staged) */
    int32_t *state;               /* long mode: [n_streams] walk state */
    int32_t *start, *end;         /* long mode: [n_chunks] the state a chunk starts / ends in (staged) */
    int T;                        /* tail letters; 0 in long mode */
    int L;
};

__device__ __forceinline__ long long chunk_stream(const StreamsArgs &a, long long h) {
    const long long s = a.ids ? (long long)__ldg(a.ids + h) : h;
    return (s >= 0 && s < a.n_streams) ? s : -1;           /* ids are validated by the caller; never index outside */
}

/* the seam of chunk h: walk tail || first min(T, n) letters from the root, report what straddles the chunk's start,
 * stage the next tail */
__global__ void __launch_bounds__(kDfaThreads) acb_seam_kernel(const __grid_constant__ ScanParams p, const StreamsArgs a) {
    const long long h = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (h >= p.n_hay) return;
    const long long s = chunk_stream(a, h);
    if (s < 0) return;
    const long long hs = hay_start(p.offsets, p.stride_bytes, h), he = hay_start(p.offsets, p.stride_bytes, h + 1);
    const int L = p.L, ls = p.letter_shift;                      /* L == 1 << ls */
    const long long n = (he - hs) >> ls;
    const long long t = min((long long)a.T, a.kept ? a.kept[s] : a.pos[s]), m = min((long long)a.T, n);
    const uint8_t *tail = a.tail + s * a.T * L, *text = p.hay + hs;
    const long long tb = t * L;
    int32_t st = 0;
    for (long long i = 0; i < (t + m) * L; ++i) {
        const uint8_t c = i < tb ? tail[i] : text[i - tb];
        const long long col = (long long)__ldg(p.cls + c) * p.S;
        int32_t nx;
        while ((nx = __ldg(p.gto + col + st)) < 0 && st != 0) st = __ldg(p.fail + st);   /* src/trie.c:182-190 */
        st = (nx < 0) ? 0 : (nx & kIdMask);
        if (i < tb || st == 0 || ((i + 1) & (L - 1))) continue;
        const long long e = ((i + 1) >> ls) - 1;                 /* letter of the seam */
        const int32_t o1 = __ldg(p.out_ptr + st + 1);
        for (int32_t o = __ldg(p.out_ptr + st); o < o1; ++o) {
            const int32_t k = __ldg(p.out_idx + o);
            if (e - __ldg(p.key_len + k) + 1 >= t) break;         /* longest first: this key and the rest start in the chunk */
            unsigned long long g = atomicAdd(p.count, 1ULL);
            if (g < (unsigned long long)p.cap) {
                acb_match r;
                r.hay_id = (int32_t)h;
                r.end_index = (int32_t)(e - t);
                r.key_id = k;
                p.out[g] = r;
            }
        }
    }
    const long long nt = min((long long)a.T, t + n), from = (t + n - nt) * L;
    uint8_t *dst = a.next_tail + h * a.T * L;
    for (long long j = 0; j < nt * L; ++j) {
        const long long x = from + j;
        dst[j] = x < tb ? tail[x] : text[x - tb];
    }
}

__global__ void acb_streams_gather_kernel(const StreamsArgs a, long long n_chunks) {
    const long long h = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (h >= n_chunks) return;
    const long long s = chunk_stream(a, h);
    a.start[h] = s < 0 ? 0 : a.state[s];
}

/* switch the fed streams to what the feed staged, only when its records fit (count == nullptr: unconditionally).
 * koff: the compacted chunks' byte offsets of a feed with a skip set */
__global__ void acb_streams_commit_kernel(const StreamsArgs a, const long long *off, long long stride, long long n_chunks,
                                          const unsigned long long *count, long long cap, const long long *koff) {
    const long long h = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (h >= n_chunks || (count && *count > (unsigned long long)cap)) return;
    const long long s = chunk_stream(a, h);
    if (s < 0) return;
    if (a.end) a.state[s] = a.end[h];
    const long long tb = (long long)a.T * a.L;
    for (long long j = 0; j < tb; ++j) a.tail[s * tb + j] = a.next_tail[h * tb + j];
    a.pos[s] += (hay_start(off, stride, h + 1) - hay_start(off, stride, h)) / a.L;
    if (a.kept) a.kept[s] += (__ldg(koff + h + 1) - __ldg(koff + h)) / a.L;
}

__global__ void acb_streams_reset_kernel(const StreamsArgs a, long long n_ids) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_ids) return;
    const long long s = chunk_stream(a, i);
    if (s < 0) return;
    a.pos[s] = 0;
    if (a.kept) a.kept[s] = 0;
    if (a.state) a.state[s] = 0;
}

/* flag[ids[i]] = 0 (the left-neighbour flags of whole-word stream batches) */
__global__ void acb_streams_clear_kernel(const int32_t *ids, long long n_ids, long long n_streams, uint8_t *flag) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_ids) return;
    const long long s = ids[i];
    if (s >= 0 && s < n_streams) flag[s] = 0;
}
} // namespace

struct acb_streams {
    int device = 0;
    int32_t L = 1, T = 0, S = 0;                 /* letter width, tail letters and (long mode) state count of the table */
    int long_mode = 0;
    long long n = 0;
    long long *d_pos = nullptr;
    uint8_t *d_tail = nullptr;
    int32_t *d_state = nullptr;
    uint8_t *d_next_tail = nullptr; size_t next_tail_cap = 0;     /* per-feed staging, grown on demand */
    int32_t *d_start = nullptr; size_t start_cap = 0;
    int32_t *d_end = nullptr; size_t end_cap = 0;
    int32_t *d_ids = nullptr; size_t ids_cap = 0;                 /* ids of a host feed or a reset, uploaded */
    std::vector<uint32_t> skip;                                   /* the skip set (find_all batches only), host copy */
    long long *d_kept = nullptr;                                  /* with a skip set: kept letters consumed per stream */
    /* leftmost-longest batches (acb_streams_new_leftmost): the tail holds the letters after X, the position up to which
     * every match is decided and emitted; d_hold[s] = pos - X of stream s (<= T).  Per-feed scratch, grown on demand. */
    int leftmost = 0;
    int kind = ACB_SELECT_LONGEST;                                /* the selection of a leftmost batch */
    long long *d_hold = nullptr;
    long long *d_soff = nullptr; size_t soff_cap = 0;             /* staged byte offsets [n_chunks + 1] */
    long long *d_aux = nullptr; size_t aux_cap = 0;               /* per chunk: last chosen end, new X, window offsets */
    uint8_t *d_stage = nullptr; size_t stage_cap = 0;             /* held || chunk, per chunk */
    uint8_t *d_win = nullptr; size_t win_cap = 0;                 /* replacing feeds: the decided windows [X, X_new) */
    long long *d_ts = nullptr; size_t ts_cap = 0;                 /* first haystack of every gather tile */
    acb_match *d_full = nullptr; size_t full_cap = 0;             /* the full list of the staged batch */
    acb_match *d_settled = nullptr; size_t settled_cap = 0;       /* ... the records that start before the frontier */
    uint8_t *d_flag = nullptr; size_t flag_cap = 0;
    acb_match *d_chosen = nullptr; size_t chosen_cap = 0;         /* replacing feeds: the chosen records */
    uint8_t *d_tmp = nullptr; size_t tmp_cap = 0;                 /* cub scratch */
    unsigned long long *d_ctr = nullptr, *h_ctr = nullptr;        /* [0] full, [1] settled, [2] chosen, [3] sizes; h_ctr pinned */
    cudaEvent_t ev[12] = {};                                      /* kernel timing, a pair per stage */
    /* whole-word batches (acb_streams_new_words; leftmost or find_all): the tail holds up to T + 1 letters, and d_left[s]
     * = 1 when the letter just before them exists and is a word letter.  The word set belongs to the batch. */
    int words = 0;
    uint8_t *d_left = nullptr;
    uint32_t *d_bits = nullptr; long long n_bits = 0;
    unsigned long long *d_keys = nullptr; size_t keys_cap = 0;    /* find_all word feeds: sort keys, 2 per kept record */
    /* case-folded batches (acb_streams_new_folded): fed with the folded table only.  The find_all feed folds the chunks
     * once, into d_fold (the device feed) or in place (the host feed's upload), and with aliases scans into d_full. */
    int fold = 0;
    uint8_t *d_fold = nullptr; size_t fold_cap = 0;
};

static int32_t tail_letters(const acb_table *tb) { return std::max<int32_t>(tb->max_key_bytes / tb->L - 1, 0); }

static int streams_check_table(const acb_streams *ss, const acb_table *tb) {
    if (tb->fold != ss->fold) {                    /* the tables can share L and T: the check below would not tell them apart */
        acb_set_error(!ss->fold ? "a stream batch does not take a case-folded table"
                      : !tb->fold ? "a case-folded stream batch takes the folded table (acb_table_upload_folded)"
                                  : "a case-folded stream batch takes a table of its own fold (ASCII or letter map)");
        return ACB_EINVAL;
    }
    if (tb->device != ss->device || tb->L != ss->L || (!ss->long_mode && tail_letters(tb) != ss->T) || (ss->long_mode && tb->S != ss->S)) {
        acb_set_error("the table does not belong to this stream batch (device %d/%d, letter bytes %d/%d, tail %d/%d, states %d/%d)",
                      tb->device, ss->device, tb->L, ss->L, ss->long_mode ? 0 : tail_letters(tb), ss->T, tb->S, ss->S);
        return ACB_EINVAL;
    }
    return ACB_OK;
}

static StreamsArgs streams_args(const acb_streams *ss, const int32_t *d_ids) {
    StreamsArgs a;
    memset(&a, 0, sizeof(a));
    a.ids = d_ids; a.n_streams = ss->n; a.pos = ss->d_pos; a.kept = ss->d_kept; a.tail = ss->d_tail; a.state = ss->d_state; a.T = ss->T; a.L = ss->L;
    return a;
}

extern "C" void acb_streams_free(acb_streams *ss) {
    DeviceRestore keep_device;
    if (!ss) return;
    cudaSetDevice(ss->device);
    cudaFree(ss->d_pos); cudaFree(ss->d_tail); cudaFree(ss->d_state); cudaFree(ss->d_next_tail);
    cudaFree(ss->d_start); cudaFree(ss->d_end); cudaFree(ss->d_ids); cudaFree(ss->d_kept);
    cudaFree(ss->d_hold); cudaFree(ss->d_soff); cudaFree(ss->d_aux); cudaFree(ss->d_stage); cudaFree(ss->d_win); cudaFree(ss->d_ts);
    cudaFree(ss->d_full); cudaFree(ss->d_settled); cudaFree(ss->d_flag); cudaFree(ss->d_chosen); cudaFree(ss->d_tmp);
    cudaFree(ss->d_ctr); cudaFree(ss->d_left); cudaFree(ss->d_bits); cudaFree(ss->d_keys); cudaFree(ss->d_fold);
    if (ss->h_ctr) cudaFreeHost(ss->h_ctr);
    for (cudaEvent_t e : ss->ev) if (e) cudaEventDestroy(e);
    delete ss;
}

/* a find_all or iter_long batch of the table's kind (folded or not); the public constructors refuse a folded table */
static int streams_new(const acb_table *tb, int64_t n_streams, int long_mode, acb_streams **out) {
    if (!tb || !out || n_streams < 0) { acb_set_error("bad argument"); return ACB_EINVAL; }
    *out = nullptr;
    if (n_streams > 0x7fffffffLL) { acb_set_error("more than 2^31-1 streams"); return ACB_ERANGE; }
    CUDA_TRY(cudaSetDevice(tb->device));
    acb_streams *ss = new (std::nothrow) acb_streams();
    if (!ss) { acb_set_error("out of memory"); return ACB_ENOMEM; }
    ss->device = tb->device; ss->L = tb->L; ss->S = tb->S; ss->long_mode = long_mode ? 1 : 0; ss->fold = tb->fold;
    ss->T = ss->long_mode ? 0 : tail_letters(tb);
    ss->n = n_streams;
    const size_t n = (size_t)std::max<int64_t>(n_streams, 1);
    cudaError_t e = cudaMalloc(reinterpret_cast<void **>(&ss->d_pos), n * sizeof(long long));
    if (e == cudaSuccess) e = cudaMemset(ss->d_pos, 0, n * sizeof(long long));
    if (e == cudaSuccess && ss->T) e = cudaMalloc(reinterpret_cast<void **>(&ss->d_tail), n * ss->T * ss->L);
    if (e == cudaSuccess && ss->long_mode) e = cudaMalloc(reinterpret_cast<void **>(&ss->d_state), n * sizeof(int32_t));
    if (e == cudaSuccess && ss->long_mode) e = cudaMemset(ss->d_state, 0, n * sizeof(int32_t));
    if (e != cudaSuccess) {
        acb_set_error("allocating %lld streams: %s", (long long)n_streams, cudaGetErrorString(e));
        acb_streams_free(ss);
        return ACB_ECUDA;
    }
    *out = ss;
    return ACB_OK;
}

extern "C" int acb_streams_new(const acb_table *tb, int64_t n_streams, int long_mode, acb_streams **out) {
    DeviceRestore keep_device;
    if (out) *out = nullptr;
    if (refuse_folded(tb, "a stream batch")) return ACB_EINVAL;
    return streams_new(tb, n_streams, long_mode, out);
}

/* A folded find_all feed's scan and seam walk (DESIGN section 4.18): the chunks folded once -- in place when `in_place`
 * (the host feed's upload, the library's own copy), else into ss->d_fold -- then the scan and the seam kernel over the
 * folded copy, so the staged tails hold folded letters (a find_all tail is only walked, never output).  Without aliases
 * the records go to p's buffer as in the plain feed.  With aliases they go to ss->d_full, grown until the full list
 * fits (one wait for its size), and are expanded into p's buffer, *p.count = the expanded total: the commit's fit test
 * then sees what the caller receives. */
static int streams_scan_folded(acb_streams *ss, acb_table *tb, ScanParams &p, StreamsArgs &a, bool in_place, unsigned grid,
                               cudaStream_t s, int algo) {
    int rc;
    const long long total = p.total;
    /* acb_scan_device's checks, before the fold: the plain feed gets the same refusals through it */
    if ((rc = check_scan_shape(tb, total, reinterpret_cast<const int64_t *>(p.offsets), p.n_hay, p.stride_bytes))) return rc;
    uint8_t *folded = const_cast<uint8_t *>(p.hay);
    if (!in_place) {
        if ((rc = ensure(&ss->d_fold, &ss->fold_cap, (size_t)total + 64))) return rc;
        folded = ss->d_fold;
    }
    if ((rc = timing_mark(&tb->f_ev[0], s)) || (rc = fold_text(tb, p.hay, folded, total, s)) || (rc = timing_mark(&tb->f_ev[1], s)) ||
        (rc = timing_ms(tb->f_ev[0], tb->f_ev[1], &g_fold_ms[0])))
        return rc;
    ScanParams q = p;
    q.hay = folded;
    if (ss->T > 0) {
        if ((rc = ensure(&ss->d_next_tail, &ss->next_tail_cap, (size_t)p.n_hay * ss->T * ss->L))) return rc;
        a.next_tail = ss->d_next_tail;
    }
    for (;;) {
        if (tb->n_alias) {
            size_t fcap = std::max<size_t>(ss->full_cap, 4096);
            if ((rc = ensure(&ss->d_full, &ss->full_cap, fcap))) return rc;
            q.out = ss->d_full;
            q.cap = (long long)std::min<size_t>(ss->full_cap, 0x7fffffffULL);
            q.count = ss->d_ctr;
            CUDA_TRY(cudaMemsetAsync(ss->d_ctr, 0, sizeof(unsigned long long), s));
        }
        if (tb->n_keys > 0 && (rc = scan_text(tb, q, total, p.n_hay, algo, s))) return rc;
        if (ss->T > 0) {
            acb_seam_kernel<<<grid, kDfaThreads, 0, s>>>(q, a);
            if ((rc = launched("seam kernel"))) return rc;
        }
        if (!tb->n_alias) return ACB_OK;
        CUDA_TRY(cudaMemcpyAsync(ss->h_ctr, ss->d_ctr, sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
        CUDA_TRY(cudaStreamSynchronize(s));
        if (ss->h_ctr[0] <= (unsigned long long)q.cap) break;
        if (ss->h_ctr[0] > 0x7fffffffULL) { acb_set_error("more than 2^31-1 matches in one feed"); return ACB_ERANGE; }
        if ((rc = ensure(&ss->d_full, &ss->full_cap, (size_t)ss->h_ctr[0]))) return rc;
    }
    return acb_expand_aliases_device(tb, ss->d_full, (int64_t)ss->h_ctr[0], p.out, p.cap, reinterpret_cast<int64_t *>(p.count), s);
}

/* the device feed; d_count is zeroed here, on `s`.  in_place: d_chunks is the library's own upload (a folded batch may
 * fold it in place) */
static int streams_feed(acb_streams *ss, acb_table *tb, const uint8_t *d_chunks, int64_t total, const int64_t *d_off,
                        int64_t n_chunks, int64_t stride, const int32_t *d_ids, acb_match *d_out, int64_t cap,
                        int64_t *d_count, cudaStream_t s, int algo, bool in_place = false) {
    if (!ss || !tb || !d_count || total < 0 || n_chunks < 0 || cap < 0 || (cap > 0 && !d_out)) { acb_set_error("bad argument"); return ACB_EINVAL; }
    if (ss->leftmost) { acb_set_error("a leftmost-longest stream batch takes acb_streams_feed_leftmost_* or acb_streams_replace_*"); return ACB_EINVAL; }
    if (ss->words) { acb_set_error("a whole-word stream batch takes acb_streams_feed_words_*"); return ACB_EINVAL; }
    int rc = streams_check_table(ss, tb);
    if (rc != ACB_OK) return rc;
    if (n_chunks > ss->n) { acb_set_error("%lld chunks for %lld streams", (long long)n_chunks, ss->n); return ACB_EINVAL; }
    if (!d_off && n_chunks && (rc = check_stride(ss->L, total, n_chunks, stride, 1))) return rc;
    if (algo == ACB_ALGO_AUTO) algo = ss->long_mode ? ACB_ALGO_LONG : ACB_ALGO_FILTER;
    if (ss->long_mode ? algo != ACB_ALGO_LONG : (algo != ACB_ALGO_FILTER && algo != ACB_ALGO_DFA)) {
        acb_set_error("algo %d does not fit a %s stream batch", algo, ss->long_mode ? "iter_long" : "find_all");
        return ACB_EINVAL;
    }
    CUDA_TRY(cudaSetDevice(ss->device));
    CUDA_TRY(cudaMemsetAsync(d_count, 0, sizeof(int64_t), s));
    if (ss->fold) g_fold_ms[0] = g_fold_ms[1] = 0.f;
    if (total == 0 || n_chunks == 0) return ACB_OK;              /* empty chunks move no stream */
    if (reinterpret_cast<uintptr_t>(d_chunks) & 15) { acb_set_error("d_chunks must be 16-byte aligned"); return ACB_EINVAL; }
    ScanParams p;
    fill_params(tb, p, d_chunks, total, d_off, n_chunks, stride, d_out, cap, d_count);
    StreamsArgs a = streams_args(ss, d_ids);
    const unsigned grid = (unsigned)((n_chunks + kDfaThreads - 1) / kDfaThreads);
    if (ss->long_mode) {
        if ((rc = ensure(&ss->d_start, &ss->start_cap, (size_t)n_chunks)) || (rc = ensure(&ss->d_end, &ss->end_cap, (size_t)n_chunks))) return rc;
        a.start = ss->d_start;
        a.end = ss->d_end;
        acb_streams_gather_kernel<<<grid, kDfaThreads, 0, s>>>(a, n_chunks);
        CUDA_TRY(cudaGetLastError());
        p.long_start = a.start;
        p.long_end = a.end;
        acb_long_kernel<<<grid, kDfaThreads, 0, s>>>(p);
        if ((rc = launched("stream iter_long kernel", 2))) return rc;
    } else if (ss->d_kept) {                                     /* skip set: compact, scan, walk the seams, map back */
        long long kept = 0;
        CompactMeta meta;
        if ((rc = compact(tb, d_chunks, total, d_off, n_chunks, stride, ss->skip.data(), (int64_t)ss->skip.size(), s, &kept, &meta))) return rc;
        const int64_t *koff = reinterpret_cast<const int64_t *>(tb->k_coff);
        if (kept && tb->n_keys > 0 && (rc = acb_scan_device(tb, tb->k_buf, kept, koff, n_chunks, 0, d_out, cap, d_count, s, algo))) return rc;
        if (ss->T > 0) {
            if ((rc = ensure(&ss->d_next_tail, &ss->next_tail_cap, (size_t)n_chunks * ss->T * ss->L))) return rc;
            ScanParams pk;
            fill_params(tb, pk, tb->k_buf, kept, koff, n_chunks, 0, d_out, cap, d_count);
            a.next_tail = ss->d_next_tail;
            acb_seam_kernel<<<grid, kDfaThreads, 0, s>>>(pk, a);
            if ((rc = launched("seam kernel"))) return rc;
        }
        if ((rc = launch_remap(tb, meta, d_off, stride, d_out, cap, d_count, s))) return rc;
    } else if (ss->fold) {
        if ((rc = streams_scan_folded(ss, tb, p, a, in_place, grid, s, algo))) return rc;
    } else {
        if (tb->n_keys > 0 && (rc = acb_scan_device(tb, d_chunks, total, d_off, n_chunks, stride, d_out, cap, d_count, s, algo))) return rc;
        if (ss->T > 0) {
            if ((rc = ensure(&ss->d_next_tail, &ss->next_tail_cap, (size_t)n_chunks * ss->T * ss->L))) return rc;
            a.next_tail = ss->d_next_tail;
            acb_seam_kernel<<<grid, kDfaThreads, 0, s>>>(p, a);
            if ((rc = launched("seam kernel"))) return rc;
        }
    }
    acb_streams_commit_kernel<<<grid, kDfaThreads, 0, s>>>(a, reinterpret_cast<const long long *>(d_off), stride, n_chunks,
                                                          reinterpret_cast<const unsigned long long *>(d_count), cap,
                                                          tb->k_coff);
    if ((rc = launched("stream commit"))) return rc;
    if (ss->d_kept && (rc = scratch_done(&tb->k_done, s))) return rc;    /* the commit read tb->k_coff */
    return ACB_OK;
}

extern "C" int acb_streams_feed_device(acb_streams *ss, acb_table *tb, const uint8_t *d_chunks, int64_t total_bytes,
                                       const int64_t *d_offsets, int64_t n_chunks, int64_t stride_bytes, const int32_t *d_ids,
                                       acb_match *d_out, int64_t cap, int64_t *d_count, void *stream, int algo) {
    DeviceRestore keep_device;
    return streams_feed(ss, tb, d_chunks, total_bytes, d_offsets, n_chunks, stride_bytes, d_ids, d_out, cap, d_count,
                        reinterpret_cast<cudaStream_t>(stream), algo);
}

/* ids of a host call: each in [0, n_streams), no two alike */
static int check_ids(const acb_streams *ss, const int32_t *ids, int64_t n) {
    std::vector<uint8_t> seen;
    try { seen.assign((size_t)ss->n, 0); } catch (const std::exception &) { acb_set_error("out of host memory"); return ACB_ENOMEM; }
    for (int64_t i = 0; i < n; i++) {
        if (ids[i] < 0 || ids[i] >= ss->n) { acb_set_error("stream id %d out of range [0, %lld)", ids[i], ss->n); return ACB_EINVAL; }
        if (seen[ids[i]]++) { acb_set_error("stream id %d given twice", ids[i]); return ACB_EINVAL; }
    }
    return ACB_OK;
}

/* the ids of a host feed, when given, to ss->d_ids on s (after the chunks and their offsets) */
static int upload_ids(acb_streams *ss, const int32_t *ids, int64_t n, cudaStream_t s) {
    if (!ids) return ACB_OK;
    int rc = ensure(&ss->d_ids, &ss->ids_cap, (size_t)n);
    if (rc != ACB_OK) return rc;
    if (n) CUDA_TRY(cudaMemcpyAsync(ss->d_ids, ids, (size_t)n * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    return ACB_OK;
}

extern "C" int acb_streams_feed_host(acb_streams *ss, acb_table *tb, const uint8_t *chunks, int64_t total_bytes,
                                     const int64_t *offsets, int64_t n_chunks, int64_t stride_bytes, const int32_t *ids,
                                     acb_match *out, int64_t cap, int64_t *n_found, int algo, int sort) {
    DeviceRestore keep_device;
    if (!ss || !tb || !n_found || total_bytes < 0 || n_chunks < 0 || cap < 0 || (total_bytes && !chunks)) { acb_set_error("bad argument"); return ACB_EINVAL; }
    *n_found = 0;
    tb->h_out_n = 0;
    if (ss->leftmost) { acb_set_error("a leftmost-longest stream batch takes acb_streams_feed_leftmost_* or acb_streams_replace_*"); return ACB_EINVAL; }
    if (ss->words) { acb_set_error("a whole-word stream batch takes acb_streams_feed_words_*"); return ACB_EINVAL; }
    int rc;
    if (ids && (rc = check_ids(ss, ids, n_chunks))) return rc;
    if ((rc = streams_check_table(ss, tb))) return rc;
    if (n_chunks > ss->n) { acb_set_error("%lld chunks for %lld streams", (long long)n_chunks, ss->n); return ACB_EINVAL; }
    if (ss->fold) g_fold_ms[0] = g_fold_ms[1] = 0.f;
    if (total_bytes == 0 || n_chunks == 0) return ACB_OK;
    const int64_t *d_off = nullptr;
    if ((rc = upload_batch(tb, chunks, total_bytes, offsets, n_chunks, &d_off)) || (rc = upload_ids(ss, ids, n_chunks, tb->stream)) ||
        (rc = ensure(&tb->w_out, &tb->w_out_cap, (size_t)std::max<int64_t>(cap, 1))))
        return rc;
    cudaStream_t s = tb->stream;
    if ((rc = streams_feed(ss, tb, tb->w_hay, total_bytes, d_off, n_chunks, stride_bytes, ids ? ss->d_ids : nullptr, tb->w_out, cap,
                           reinterpret_cast<int64_t *>(tb->w_count), s, algo, true)))
        return rc;
    return read_back(tb, tb->w_count, tb->w_out, cap, sort, n_chunks, (offsets ? total_bytes : stride_bytes) / tb->L, out, n_found, s);
}

extern "C" int acb_streams_reset(acb_streams *ss, const int32_t *ids, int64_t n) {
    DeviceRestore keep_device;
    if (!ss || n < 0) { acb_set_error("bad argument"); return ACB_EINVAL; }
    int rc;
    if (ids && (rc = check_ids(ss, ids, n))) return rc;
    CUDA_TRY(cudaSetDevice(ss->device));
    CUDA_TRY(cudaDeviceSynchronize());                           /* feeds in flight on any stream see the old state */
    if (!ids) {
        CUDA_TRY(cudaMemset(ss->d_pos, 0, (size_t)std::max<long long>(ss->n, 1) * sizeof(long long)));
        if (ss->d_kept) CUDA_TRY(cudaMemset(ss->d_kept, 0, (size_t)std::max<long long>(ss->n, 1) * sizeof(long long)));
        if (ss->d_state) CUDA_TRY(cudaMemset(ss->d_state, 0, (size_t)std::max<long long>(ss->n, 1) * sizeof(int32_t)));
    } else if (n) {
        if ((rc = ensure(&ss->d_ids, &ss->ids_cap, (size_t)n))) return rc;
        CUDA_TRY(cudaMemcpy(ss->d_ids, ids, (size_t)n * sizeof(int32_t), cudaMemcpyHostToDevice));
        StreamsArgs a = streams_args(ss, ss->d_ids);
        if (ss->d_hold) a.kept = ss->d_hold;                     /* leftmost (no skip set): nothing held back either */
        acb_streams_reset_kernel<<<(unsigned)((n + 255) / 256), 256>>>(a, n);
        if ((rc = launched("stream reset"))) return rc;
        if (ss->d_left) {                                        /* whole words: no letter before the start */
            acb_streams_clear_kernel<<<(unsigned)((n + 255) / 256), 256>>>(ss->d_ids, n, ss->n, ss->d_left);
            if ((rc = launched("stream reset"))) return rc;
        }
    }
    if (!ids && ss->d_hold) CUDA_TRY(cudaMemset(ss->d_hold, 0, (size_t)std::max<long long>(ss->n, 1) * sizeof(long long)));
    if (!ids && ss->d_left) CUDA_TRY(cudaMemset(ss->d_left, 0, (size_t)std::max<long long>(ss->n, 1)));
    CUDA_TRY(cudaDeviceSynchronize());
    return ACB_OK;
}

extern "C" int acb_streams_positions(acb_streams *ss, int64_t *out, int64_t cap) {
    DeviceRestore keep_device;
    if (!ss || cap < ss->n || (ss->n && !out)) { acb_set_error("bad argument (capacity %lld for %lld streams)", (long long)cap, ss ? ss->n : 0LL); return ACB_EINVAL; }
    CUDA_TRY(cudaSetDevice(ss->device));
    CUDA_TRY(cudaDeviceSynchronize());
    if (ss->n) CUDA_TRY(cudaMemcpy(out, ss->d_pos, (size_t)ss->n * sizeof(long long), cudaMemcpyDeviceToHost));
    return ACB_OK;
}

extern "C" int acb_streams_new_skip(const acb_table *tb, int64_t n_streams, const uint32_t *skip, int64_t n_skip, acb_streams **out) {
    DeviceRestore keep_device;
    if (!tb || !out) { acb_set_error("bad argument"); return ACB_EINVAL; }
    *out = nullptr;
    int rc = check_skip(skip, n_skip, ACB_ALGO_FILTER);
    if (rc != ACB_OK) return rc;
    CUDA_TRY(cudaSetDevice(tb->device));                    /* for the allocation below: acb_streams_new restores it */
    if ((rc = acb_streams_new(tb, n_streams, 0, out))) return rc;
    acb_streams *ss = *out;
    const size_t n = (size_t)std::max<int64_t>(n_streams, 1);
    try {
        ss->skip.assign(skip, skip + n_skip);
    } catch (const std::exception &) {
        acb_streams_free(ss);
        *out = nullptr;
        acb_set_error("out of host memory");
        return ACB_ENOMEM;
    }
    cudaError_t e = cudaMalloc(reinterpret_cast<void **>(&ss->d_kept), n * sizeof(long long));
    if (e == cudaSuccess) e = cudaMemset(ss->d_kept, 0, n * sizeof(long long));
    if (e != cudaSuccess) {
        acb_set_error("allocating %lld streams: %s", (long long)n_streams, cudaGetErrorString(e));
        acb_streams_free(ss);
        *out = nullptr;
        return ACB_ECUDA;
    }
    return ACB_OK;
}

/* ------------------------------------------------------------ dictionary lookups */
/* exists / match / longest_prefix / get for a whole batch of keys (trie_find / trie_longest, src/trie.c:139-174): one
 * lane per query walks the trie edges of the flattened table from the root, byte by byte, and stops at the first
 * missing edge.  Flattening keeps only nodes with a live key below them, so the walk takes exactly the edges the host
 * trie's walk takes.  Every step is a dependent load from the goto table (gigabytes for a million keys): the kernel is
 * bound by the latency of those loads, so it only keeps the byte classes in shared memory and many lanes in flight. */
namespace {
constexpr int kLookupThreads = 256;

struct LookupParams {
    const uint8_t *keys;
    const long long *offsets;      /* nullptr => fixed stride */
    long long n, stride;
    const uint8_t *cls;
    const int32_t *gto;            /* flagged goto (kTermBit) */
    const int32_t *key_of;
    long long S;
    int32_t letter_shift;
    int32_t *key_id, *prefix;
};

/* one byte of the dictionary walks: the child of state s along `byte`, or -1.  Class 0 needs no test: its column is all
 * -1 unless K == 256, when it is a real byte.  The goto table can pass 2^31 entries, hence the 64-bit index. */
__device__ __forceinline__ int32_t trie_step(const int32_t *gto, const uint8_t *cls, long long S, uint8_t byte, int32_t s) {
    const int32_t nx = __ldg(gto + (long long)cls[byte] * S + s);
    return nx < 0 ? -1 : (nx & kIdMask);           /* drop kTermBit */
}

__global__ void __launch_bounds__(kLookupThreads) acb_lookup_kernel(const __grid_constant__ LookupParams p) {
    __shared__ uint8_t cls[256];
    for (int i = threadIdx.x; i < 256; i += blockDim.x) cls[i] = p.cls[i];
    __syncthreads();
    for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < p.n; q += (long long)gridDim.x * blockDim.x) {
        const long long b0 = p.offsets ? __ldg(p.offsets + q) : q * p.stride;
        const long long b1 = p.offsets ? __ldg(p.offsets + q + 1) : b0 + p.stride;
        int32_t s = 0;
        long long i = b0;
        for (; i < b1; ++i) {
            const int32_t nx = trie_step(p.gto, cls, p.S, __ldg(p.keys + i), s);
            if (nx < 0) break;
            s = nx;
        }
        p.key_id[q] = (i == b1 && b1 > b0) ? __ldg(p.key_of + s) : -1;
        p.prefix[q] = (int32_t)((i - b0) >> p.letter_shift);   /* whole letters only; at most the longest key */
    }
}
} // namespace

extern "C" int acb_lookup_device(acb_table *tb, const uint8_t *d_keys, int64_t total_bytes, const int64_t *d_offsets,
                                 int64_t n_keys, int64_t stride_bytes, int32_t *d_key_id, int32_t *d_prefix, void *stream) {
    DeviceRestore keep_device;
    if (refuse_folded(tb, "a lookup")) return ACB_EINVAL;
    if (!tb || total_bytes < 0 || n_keys < 0 || (total_bytes && !d_keys) || (n_keys && (!d_key_id || !d_prefix))) {
        acb_set_error("bad argument");
        return ACB_EINVAL;
    }
    int rc;
    if (!d_offsets && (rc = check_stride(tb->L, total_bytes, n_keys, stride_bytes, 0))) return rc;
    if (n_keys == 0) return ACB_OK;
    CUDA_TRY(cudaSetDevice(tb->device));
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    LookupParams p;
    p.keys = d_keys; p.offsets = reinterpret_cast<const long long *>(d_offsets); p.n = n_keys; p.stride = stride_bytes;
    p.cls = tb->d_cls; p.gto = tb->d_goto; p.key_of = tb->d_keyof; p.S = tb->S;
    p.letter_shift = tb->L == 4 ? 2 : (tb->L == 2 ? 1 : 0);
    p.key_id = d_key_id; p.prefix = d_prefix;
    const long long grid = std::min<long long>((n_keys + kLookupThreads - 1) / kLookupThreads, grid_sms(tb) * 8);
    if ((rc = timing_mark(&tb->ev0, s))) return rc;
    acb_lookup_kernel<<<(unsigned)grid, kLookupThreads, 0, s>>>(p);
    if ((rc = launched("lookup kernel")) || (rc = timing_mark(&tb->ev1, s))) return rc;
    return timing_ms(tb->ev0, tb->ev1, &g_last_ms);
}

extern "C" int acb_lookup_host(acb_table *tb, const uint8_t *keys, int64_t total_bytes, const int64_t *offsets,
                               int64_t n_keys, int64_t stride_bytes, int32_t *key_id, int32_t *prefix) {
    DeviceRestore keep_device;
    if (refuse_folded(tb, "a lookup")) return ACB_EINVAL;
    if (!tb || total_bytes < 0 || n_keys < 0 || (total_bytes && !keys) || (n_keys && (!key_id || !prefix))) {
        acb_set_error("bad argument");
        return ACB_EINVAL;
    }
    CUDA_TRY(cudaSetDevice(tb->device));
    int rc = offsets ? check_offsets(tb->L, offsets, n_keys, total_bytes) : check_stride(tb->L, total_bytes, n_keys, stride_bytes, 0);
    if (rc != ACB_OK) return rc;
    if (n_keys == 0) return ACB_OK;
    const int64_t *d_off = nullptr;
    if ((rc = upload_batch(tb, keys, total_bytes, offsets, n_keys, &d_off)) || (rc = ensure(&tb->w_lk, &tb->w_lk_cap, 2 * (size_t)n_keys))) return rc;
    cudaStream_t s = tb->stream;
    if ((rc = acb_lookup_device(tb, tb->w_hay, total_bytes, d_off, n_keys, stride_bytes, tb->w_lk, tb->w_lk + n_keys, s))) return rc;
    CUDA_TRY(cudaMemcpyAsync(key_id, tb->w_lk, (size_t)n_keys * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaMemcpyAsync(prefix, tb->w_lk + n_keys, (size_t)n_keys * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    return ACB_OK;
}

/* ------------------------------------------------------------ dictionary selection */
/* keys / values / items (prefix, wildcard, how) for a whole batch of patterns (src/AutomatonItemsIter.c:125-288).  The
 * reference walks the trie under the pattern with a stack, youngest child first.  In that pre-order the keys at or
 * under a node are one run of the key order, order[lo[s] .. lo[s] + cnt[s]), and a node's letter-children sorted by lo
 * are the order its stack pops them (acb_trie_key_ranges).  One lane per pattern:
 *  - without a wildcard the query is one walk down the goto table and one run;
 *  - with one, the lane walks the tree of nodes the pattern can reach depth first, taking the children of a wildcard
 *    letter from the child list.  It emits keys in rank order, so no sort is needed.
 * The walk is driven by a rank cursor r (every key of rank < r is dealt with).  At every node the lane takes the first
 * child that can still match and whose run ends after r: the goto child for a plain letter, a binary search by lo in
 * the child list for a wildcard.  A node without one is done; r moves to the end of its run and the lane goes back to
 * its parent.  The lane keeps the last kSelectPath nodes of its path; a deeper parent is found again by the same
 * descent from the deepest one kept, since the cursor leads it to the same node.  So there is no limit on the length
 * of a pattern or on its wildcard letters. */
namespace {
constexpr int kSelectThreads = 128;
constexpr int kSelectPath = 16;

struct SelectParams {
    const uint8_t *pat;
    const long long *offsets;      /* nullptr => fixed stride */
    long long n, stride;
    const uint8_t *cls;
    const int32_t *gto;            /* flagged goto (kTermBit) */
    long long S;
    const int32_t *key_of, *order, *lo, *cnt, *child_ptr, *child;
    long long wildcard;            /* letter value, -1: none */
    int32_t how, L;
    long long *out_off;            /* pass 1: the count of pattern q goes to [q + 1]; pass 2: its slice starts at [q] */
    int32_t *key_id;
    const long long *total;        /* pass 2 writes nothing when *total > cap */
    long long cap;
};

/* the state one whole letter below s, or -1 */
__device__ __forceinline__ int32_t select_letter(const SelectParams &p, const uint8_t *cls, const uint8_t *b, int32_t s) {
    for (int d = 0; d < p.L && s >= 0; ++d) s = trie_step(p.gto, cls, p.S, __ldg(b + d), s);
    return s;
}

/* the keys of one pattern of m letters at pat: counted, or (kWrite) their ids written to out; returns the count */
template <bool kWrite>
__device__ long long select_walk(const SelectParams &p, const uint8_t *cls, const uint8_t *pat, long long m, int32_t *out) {
    long long n_out = 0;
    auto emit = [&](int32_t r0, int32_t r1) {                  /* the keys of ranks r0 .. r1 */
        if (kWrite)
            for (int32_t r = r0; r < r1; ++r) out[n_out + (r - r0)] = __ldg(p.order + r);
        n_out += r1 - r0;
    };
    if (p.wildcard < 0) {                                      /* every key that starts with the pattern */
        int32_t x = 0;
        for (long long j = 0; j < m && x >= 0; ++j) x = select_letter(p, cls, pat + j * p.L, x);
        if (x >= 0) {
            const int32_t xlo = __ldg(p.lo + x);
            emit(xlo, xlo + __ldg(p.cnt + x));
        }
        return n_out;
    }
    int32_t path[kSelectPath];                                 /* path[j]: the node at depth j, for j < kSelectPath */
    path[0] = 0;
    int32_t x = 0, r = 0;
    long long j = 0;
    for (;;) {
        const int32_t xlo = __ldg(p.lo + x), xend = xlo + __ldg(p.cnt + x);
        /* the node's own key has rank xlo; ranks below r were emitted or rejected before */
        if (j > 0 && xlo >= r && (p.how == ACB_MATCH_AT_MOST_PREFIX || (p.how == ACB_MATCH_EXACT_LENGTH && j == m)) &&
            __ldg(p.key_of + x) >= 0) {
            emit(xlo, xlo + 1);
            r = xlo + 1;
        }
        int32_t c = -1;
        if (j == m) {
            if (p.how == ACB_MATCH_AT_LEAST_PREFIX) emit(max(r, xlo), xend);
        } else {
            const uint8_t *b = pat + j * p.L;
            uint32_t letter = 0;
            for (int d = 0; d < p.L; ++d) letter |= (uint32_t)__ldg(b + d) << (8 * d);
            if ((long long)letter == p.wildcard) {             /* the first child whose run ends after r */
                const int32_t c0 = __ldg(p.child_ptr + x), c1 = __ldg(p.child_ptr + x + 1);
                int32_t a = c0, z = c1;                        /* a: the first child with lo > r */
                while (a < z) {
                    const int32_t mid = (a + z) >> 1;
                    if (__ldg(p.lo + __ldg(p.child + mid)) > r) z = mid; else a = mid + 1;
                }
                if (a > c0) {
                    const int32_t y = __ldg(p.child + a - 1);
                    if (__ldg(p.lo + y) + __ldg(p.cnt + y) > r) c = y;
                }
                if (c < 0 && a < c1) c = __ldg(p.child + a);
            } else {                                           /* a letter walked in part matches nothing */
                c = select_letter(p, cls, b, x);
                if (c >= 0 && __ldg(p.lo + c) + __ldg(p.cnt + c) <= r) c = -1;
            }
        }
        if (c < 0) {                                           /* x is done: back to its parent */
            r = max(r, xend);
            if (j == 0) break;
            j = min(j - 1, (long long)kSelectPath - 1);
            x = path[j];
            continue;
        }
        x = c;
        if (++j < kSelectPath) path[j] = x;
    }
    return n_out;
}

template <bool kWrite>
__global__ void __launch_bounds__(kSelectThreads) acb_select_kernel(const __grid_constant__ SelectParams p) {
    __shared__ uint8_t cls[256];
    for (int i = threadIdx.x; i < 256; i += blockDim.x) cls[i] = p.cls[i];
    __syncthreads();
    if (kWrite && *p.total > p.cap) return;
    for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < p.n; q += (long long)gridDim.x * blockDim.x) {
        const long long b0 = p.offsets ? __ldg(p.offsets + q) : q * p.stride;
        const long long b1 = p.offsets ? __ldg(p.offsets + q + 1) : b0 + p.stride;
        const long long m = (b1 - b0) / p.L;
        if (kWrite) select_walk<true>(p, cls, p.pat + b0, m, p.key_id + p.out_off[q]);
        else p.out_off[q + 1] = select_walk<false>(p, cls, p.pat + b0, m, nullptr);
    }
}
} // namespace

extern "C" int acb_table_upload_key_ranges(acb_table *tb, const acb_trie *t) {
    DeviceRestore keep_device;
    if (!tb || !t) { acb_set_error("bad argument"); return ACB_EINVAL; }
    if (refuse_folded(tb, "a key selection")) return ACB_EINVAL;
    if (tb->d_order) return ACB_OK;
    acb_flat_view f;
    int rc = acb_trie_flat_view(t, &f);
    if (rc != ACB_OK) return rc;
    if (f.n_states != tb->S || f.n_keys != tb->n_keys || f.letter_bytes != tb->L) {
        acb_set_error("the trie is not the one this table was uploaded from");
        return ACB_EINVAL;
    }
    const size_t S = (size_t)f.n_states, n_live = (size_t)acb_trie_count(t);
    std::vector<int32_t> order, lo, cnt, child_ptr, child;
    try {
        order.resize(std::max<size_t>(n_live, 1)); lo.resize(S); cnt.resize(S); child_ptr.resize(S + 1); child.resize(S);
    } catch (const std::exception &) {
        acb_set_error("out of host memory while staging the key ranges");
        return ACB_ENOMEM;
    }
    int64_t n_edges = 0;
    if ((rc = acb_trie_key_ranges(t, order.data(), lo.data(), cnt.data(), child_ptr.data(), child.data(), &n_edges))) return rc;
    CUDA_TRY(cudaSetDevice(tb->device));
    do {
        if ((rc = upload(&tb->d_lo, lo.data(), S, tb->dev_bytes))) break;
        if ((rc = upload(&tb->d_cnt, cnt.data(), S, tb->dev_bytes))) break;
        if ((rc = upload(&tb->d_child_ptr, child_ptr.data(), S + 1, tb->dev_bytes))) break;
        if ((rc = upload(&tb->d_child, child.data(), (size_t)n_edges, tb->dev_bytes))) break;
        rc = upload(&tb->d_order, order.data(), n_live, tb->dev_bytes);   /* last: it marks the view complete */
    } while (0);
    if (rc != ACB_OK) {
        cudaFree(tb->d_lo); cudaFree(tb->d_cnt); cudaFree(tb->d_child_ptr); cudaFree(tb->d_child); cudaFree(tb->d_order);
        tb->d_lo = tb->d_cnt = tb->d_child_ptr = tb->d_child = tb->d_order = nullptr;
    }
    return rc;
}

static int select_args_ok(const acb_table *tb, int64_t wildcard, int how) {
    if (how != ACB_MATCH_EXACT_LENGTH && how != ACB_MATCH_AT_MOST_PREFIX && how != ACB_MATCH_AT_LEAST_PREFIX) {
        acb_set_error("how must be ACB_MATCH_EXACT_LENGTH, ACB_MATCH_AT_MOST_PREFIX or ACB_MATCH_AT_LEAST_PREFIX");
        return ACB_EINVAL;
    }
    if (wildcard < -1 || wildcard >= ((int64_t)1 << (8 * tb->L))) {
        acb_set_error("wildcard must be -1 or a %d-byte letter value", tb->L);
        return ACB_EINVAL;
    }
    return ACB_OK;
}

static void fill_select_params(const acb_table *tb, SelectParams &p, const uint8_t *d_pat, const int64_t *d_offsets,
                               int64_t n, int64_t stride, int64_t wildcard, int how, int64_t *d_out_off,
                               int32_t *d_key_id, int64_t cap, const int64_t *d_total) {
    p.pat = d_pat; p.offsets = reinterpret_cast<const long long *>(d_offsets); p.n = n; p.stride = stride;
    p.cls = tb->d_cls; p.gto = tb->d_goto; p.S = tb->S;
    p.key_of = tb->d_keyof; p.order = tb->d_order; p.lo = tb->d_lo; p.cnt = tb->d_cnt;
    p.child_ptr = tb->d_child_ptr; p.child = tb->d_child;
    p.wildcard = wildcard; p.how = how; p.L = tb->L;
    p.out_off = reinterpret_cast<long long *>(d_out_off); p.key_id = d_key_id;
    p.total = reinterpret_cast<const long long *>(d_total); p.cap = cap;
}

/* pass 1 and the scan: d_out_off[0..n] and *d_total, on s */
static int select_count(acb_table *tb, const SelectParams &p, int64_t n, int64_t *d_out_off, int64_t *d_total, cudaStream_t s) {
    CUDA_TRY(cudaMemsetAsync(d_out_off, 0, sizeof(int64_t), s));
    if (n == 0) {
        CUDA_TRY(cudaMemsetAsync(d_total, 0, sizeof(int64_t), s));
        return ACB_OK;
    }
    acb_select_kernel<false><<<blocks(tb, n, kSelectThreads), kSelectThreads, 0, s>>>(p);
    int rc = launched("select kernel");
    if (rc != ACB_OK) return rc;
    long long *cnt = reinterpret_cast<long long *>(d_out_off) + 1;     /* in place: counts -> inclusive sums */
    size_t temp = 0;
    CUDA_TRY(cub::DeviceScan::InclusiveSum(nullptr, temp, cnt, cnt, (long long)n, s));
    if ((rc = ensure(&tb->w_scan, &tb->w_scan_cap, temp))) return rc;
    CUDA_TRY(cub::DeviceScan::InclusiveSum(tb->w_scan, temp, cnt, cnt, (long long)n, s));
    CUDA_TRY(cudaMemcpyAsync(d_total, d_out_off + n, sizeof(int64_t), cudaMemcpyDeviceToDevice, s));
    return ACB_OK;
}

/* pass 2: the ids, when *p.total <= p.cap */
static int select_fill(acb_table *tb, const SelectParams &p, int64_t n, cudaStream_t s) {
    if (n == 0 || p.cap == 0) return ACB_OK;
    acb_select_kernel<true><<<blocks(tb, n, kSelectThreads), kSelectThreads, 0, s>>>(p);
    return launched("select kernel");
}

static int select_common_checks(const acb_table *tb, const void *pat, int64_t total_bytes, int64_t n, const void *out_off,
                                const void *key_id, int64_t cap, const void *total, int64_t wildcard, int how) {
    if (refuse_folded(tb, "a key selection")) return ACB_EINVAL;
    if (!tb || total_bytes < 0 || n < 0 || (total_bytes && !pat) || !out_off || !total || cap < 0 || (cap && !key_id)) {
        acb_set_error("bad argument");
        return ACB_EINVAL;
    }
    return select_args_ok(tb, wildcard, how);
}

static int select_view_ok(const acb_table *tb) {
    if (tb->d_order) return ACB_OK;
    acb_set_error("the key ranges are not on the device yet (acb_table_upload_key_ranges)");
    return ACB_ESTATE;
}

extern "C" int acb_select_device(acb_table *tb, const uint8_t *d_patterns, int64_t total_bytes, const int64_t *d_offsets,
                                 int64_t n, int64_t stride_bytes, int64_t wildcard, int how, int64_t *d_out_offsets,
                                 int32_t *d_key_id, int64_t cap, int64_t *d_total, void *stream) {
    DeviceRestore keep_device;
    int rc = select_common_checks(tb, d_patterns, total_bytes, n, d_out_offsets, d_key_id, cap, d_total, wildcard, how);
    if (rc != ACB_OK) return rc;
    if (!d_offsets && (rc = check_stride(tb->L, total_bytes, n, stride_bytes, 0))) return rc;
    if ((rc = select_view_ok(tb))) return rc;
    CUDA_TRY(cudaSetDevice(tb->device));
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    SelectParams p;
    fill_select_params(tb, p, d_patterns, d_offsets, n, stride_bytes, wildcard, how, d_out_offsets, d_key_id, cap, d_total);
    if ((rc = timing_mark(&tb->ev0, s)) || (rc = select_count(tb, p, n, d_out_offsets, d_total, s)) || (rc = select_fill(tb, p, n, s)) ||
        (rc = timing_mark(&tb->ev1, s)))
        return rc;
    return timing_ms(tb->ev0, tb->ev1, &g_last_ms);
}

extern "C" int acb_select_host(acb_table *tb, const uint8_t *patterns, int64_t total_bytes, const int64_t *offsets,
                               int64_t n, int64_t stride_bytes, int64_t wildcard, int how, int64_t *out_offsets,
                               int32_t *key_id, int64_t cap, int64_t *total) {
    DeviceRestore keep_device;
    int rc = select_common_checks(tb, patterns, total_bytes, n, out_offsets, key_id, cap, total, wildcard, how);
    if (rc != ACB_OK) return rc;
    if ((rc = offsets ? check_offsets(tb->L, offsets, n, total_bytes) : check_stride(tb->L, total_bytes, n, stride_bytes, 0))) return rc;
    if ((rc = select_view_ok(tb))) return rc;
    const int64_t *d_off = nullptr;
    if ((rc = upload_batch(tb, patterns, total_bytes, offsets, n, &d_off)) || (rc = ensure(&tb->w_sel_off, &tb->w_sel_off_cap, (size_t)n + 2))) return rc;
    cudaStream_t s = tb->stream;
    int64_t *d_out = reinterpret_cast<int64_t *>(tb->w_sel_off), *d_total = d_out + n + 1;
    SelectParams p;
    fill_select_params(tb, p, tb->w_hay, d_off, n, stride_bytes, wildcard, how, d_out, nullptr, 0, d_total);
    if ((rc = select_count(tb, p, n, d_out, d_total, s))) return rc;
    CUDA_TRY(cudaMemcpyAsync(out_offsets, d_out, (size_t)(n + 1) * sizeof(int64_t), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    *total = out_offsets[n];
    if (*total > cap) {
        acb_set_error("select: room for %lld ids, %lld selected", (long long)cap, (long long)*total);
        return ACB_EOVERFLOW;
    }
    if (*total == 0) return ACB_OK;
    if ((rc = ensure(&tb->w_sel_id, &tb->w_sel_id_cap, (size_t)*total))) return rc;
    p.key_id = tb->w_sel_id;
    p.cap = *total;
    if ((rc = select_fill(tb, p, n, s))) return rc;
    CUDA_TRY(cudaMemcpyAsync(key_id, tb->w_sel_id, (size_t)*total * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    return ACB_OK;
}

/* ------------------------------------------------------------ leftmost-longest selection */
/* Leftmost-longest non-overlapping matches (p = 0; take the smallest start >= p, the longest match there, continue after
 * it) are a function of the full match list alone, so they are selected from the records a scan left, in five
 * data-parallel steps: (1) radix sort by hay | start | (max_len - len); (2) the first record of every (hay, start) run is
 * the longest match starting there: a candidate, compacted with DeviceSelect; (3) next[i] = the first candidate of the
 * same haystack that starts at or after the end of candidate i (a binary search over the next len_i candidates);
 * (4) a candidate is chosen iff it lies on the next-chain from its haystack's first candidate: acb_ll_chain_kernel
 * below; (5) the chosen candidates, already in the final order, are stream-compacted into the caller's buffer. */
namespace {
constexpr int kLlTile = 2048;                             /* candidates per chain tile */
constexpr int kLlThreads = 256;
thread_local float g_ll_ms[5] = {};                       /* kernel timing: sort, candidates, successor, chain, emit */

__device__ __forceinline__ long long ll_start(const acb_match &m, const int32_t *key_len) {
    return (long long)m.end_index - __ldg(key_len + m.key_id) + 1;
}

/* flag[i] = 1 for the first record of every (hay, start) run of the sorted list */
__global__ void acb_ll_cand_kernel(const acb_match *rec, long long n, const int32_t *key_len, uint8_t *flag) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const acb_match m = rec[i];
        bool first = i == 0;
        if (!first) {
            const acb_match q = rec[i - 1];
            first = q.hay_id != m.hay_id || ll_start(q, key_len) != ll_start(m, key_len);
        }
        flag[i] = first;
    }
}

/* next[i]: the first candidate of the same haystack with start >= start_i + len_i, or -1.  A haystack's candidates have
 * distinct ascending starts, so candidate i + len_i (when it is of the same haystack) already qualifies: the search
 * covers [i + 1, i + len_i]. */
__global__ void acb_ll_next_kernel(const acb_match *cand, const unsigned long long *d_m, const int32_t *key_len, int32_t *nxt) {
    const long long M = (long long)*d_m;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < M; i += (long long)gridDim.x * blockDim.x) {
        const acb_match c = cand[i];
        const long long target = (long long)c.end_index + 1;
        long long lo = i + 1, hi = min(M, i + __ldg(key_len + c.key_id) + 1);
        while (lo < hi) {
            const long long mid = (lo + hi) >> 1;
            const acb_match q = cand[mid];
            if (q.hay_id != c.hay_id || ll_start(q, key_len) >= target) hi = mid; else lo = mid + 1;
        }
        bool ok = false;
        if (lo < M) { const acb_match q = cand[lo]; ok = q.hay_id == c.hay_id && ll_start(q, key_len) >= target; }
        nxt[i] = ok ? (int32_t)lo : -1;
    }
}

/* Chain marking over tiles of kLlTile candidates, one block per tile, tiles claimed in order from a counter.
 *  - The speculative walk (one thread, shared memory): from the tile's first candidate and from every haystack's first
 *    candidate in the tile, the chain through next[].  Every haystack that starts in the tile is exact; only the one
 *    continuing from the previous tile (candidates [0, fh)) depends on the entry the previous tile hands over.
 *  - The exit (the chain's first candidate past the tile, or -1) is published to status[t] as soon as it is known.  It
 *    does not depend on the entry when a haystack starts in the tile, or when the tile holds at least W = longest_word
 *    candidates and the chain from each of the first W joins the speculative chain inside the tile: the entry is the
 *    successor of a candidate of an earlier tile, so it lies among the first W candidates, and chains that meet stay
 *    together.  Otherwise the tile publishes after its entry is known.
 *  - The entry comes from status[t - 1] (a look-back of one tile: every tile publishes its exit itself).  The tile walks
 *    from it until it lands on the speculative chain; the speculative nodes before that point are dropped. */
__global__ void __launch_bounds__(kLlThreads) acb_ll_chain_kernel(const acb_match *cand, const unsigned long long *d_m,
                                                                  const int32_t *nxt, int W, unsigned long long *ctr,
                                                                  unsigned long long *status, uint8_t *chosen, int32_t *pos) {
    __shared__ int32_t s_next[kLlTile];
    __shared__ int32_t s_hay[kLlTile + 1];                 /* s_hay[j] = hay of candidate base + j - 1 */
    __shared__ uint8_t s_spec[kLlTile], s_fin[kLlTile];
    __shared__ long long s_tile, s_exit;
    __shared__ int s_fh;
    __shared__ volatile int s_dep;
    if (threadIdx.x == 0) s_tile = (long long)atomicAdd(ctr, 1ULL);   /* in claim order: every earlier tile is running or done */
    __syncthreads();
    const long long M = (long long)*d_m, t = s_tile, base = t * kLlTile;
    if (base >= M) return;
    const int n_tile = (int)min((long long)kLlTile, M - base);
    for (int j = threadIdx.x; j <= n_tile; j += kLlThreads) {
        s_hay[j] = base + j - 1 < 0 ? -1 : cand[base + j - 1].hay_id;
        if (j < n_tile) s_next[j] = nxt[base + j];
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        long long want = base;
        int fh = n_tile;
        for (int j = 0; j < n_tile; j++) {
            if (s_hay[j + 1] != s_hay[j]) { want = base + j; if (fh == n_tile) fh = j; }
            const bool on = want == base + j;
            s_spec[j] = on;
            if (on) want = s_next[j];
        }
        s_exit = want;
        s_fh = fh;
        s_dep = fh == n_tile && n_tile < W;
    }
    __syncthreads();
    const int fh = s_fh;
    const long long spec_exit = s_exit;
    for (int j = threadIdx.x; j < n_tile; j += kLlThreads) s_fin[j] = s_spec[j];
    if (fh == n_tile && !s_dep) {                          /* one haystack fills the tile: does every possible entry join? */
        for (int j = threadIdx.x; j < W; j += kLlThreads) {
            long long e = base + j;
            while (e >= base && e < base + n_tile && !s_spec[e - base] && !s_dep) e = s_next[e - base];
            const bool joined = e >= base && e < base + n_tile && s_spec[e - base];
            if (!joined && e != spec_exit) s_dep = 1;
        }
    }
    __syncthreads();
    const bool indep = !s_dep;
    if (threadIdx.x == 0) {
        if (indep) atomicExch(status + t, (unsigned long long)(spec_exit + 2));
        long long entry = base, exit = spec_exit;
        if (fh > 0 && t > 0) {
            unsigned long long st;
            while ((st = *reinterpret_cast<volatile unsigned long long *>(status + t - 1)) == 0) {}
            entry = (long long)st - 2;
        }
        if (entry != base) {                               /* merge on entry */
            long long e = entry;
            while (e >= base && e < base + fh && !s_spec[e - base]) { s_fin[e - base] = 1; e = s_next[e - base]; }
            const bool joined = e >= base && e < base + fh;
            const long long stop = joined ? e : base + fh;
            for (long long q = base; q >= base && q < stop; q = s_next[q - base]) s_fin[q - base] = 0;
            if (fh == n_tile && !joined) exit = e;
        }
        if (!indep) atomicExch(status + t, (unsigned long long)(exit + 2));
    }
    __syncthreads();
    for (int j = threadIdx.x; j < n_tile; j += kLlThreads) {
        chosen[base + j] = s_fin[j];
        pos[base + j] = s_fin[j];
    }
}

/* the chosen candidates (pos: their exclusive prefix count) to out[*count + pos], those past cap counted, not stored */
__global__ void acb_ll_emit_kernel(const acb_match *cand, const unsigned long long *d_m, const uint8_t *chosen, const int32_t *pos,
                                   acb_match *out, long long cap, const unsigned long long *count) {
    const long long M = (long long)*d_m;
    const unsigned long long first = *count;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < M; i += (long long)gridDim.x * blockDim.x) {
        if (!chosen[i]) continue;
        const unsigned long long p = first + (unsigned long long)pos[i];
        if (p < (unsigned long long)cap) out[p] = cand[i];
    }
}

__global__ void acb_ll_count_kernel(const unsigned long long *d_m, const uint8_t *chosen, const int32_t *pos, unsigned long long *count) {
    const long long M = (long long)*d_m;
    if (M > 0) *count += (unsigned long long)pos[M - 1] + chosen[M - 1];
}
} // namespace

/* The flagged ones of the first *d_m (<= n) records of rec, in order, to d_out[*d_count ..] (those past cap counted, not
 * stored), and *d_count += their number.  pos holds the flags and becomes their exclusive sum; tmp: cub scratch of temp
 * bytes for it. */
static int emit_flagged(acb_table *tb, const acb_match *rec, const unsigned long long *d_m, const uint8_t *flag, int32_t *pos, int n,
                        void *tmp, size_t temp, acb_match *d_out, int64_t cap, int64_t *d_count, cudaStream_t s, const char *what) {
    CUDA_TRY(cub::DeviceScan::ExclusiveSum(tmp, temp, pos, pos, n, s));
    acb_ll_emit_kernel<<<blocks(tb, n), 256, 0, s>>>(rec, d_m, flag, pos, d_out, cap, reinterpret_cast<const unsigned long long *>(d_count));
    CUDA_TRY(cudaGetLastError());
    acb_ll_count_kernel<<<1, 1, 0, s>>>(d_m, flag, pos, reinterpret_cast<unsigned long long *>(d_count));
    return launched(what, 2);
}

extern "C" int acb_last_leftmost_ms(float *ms, int32_t n) {
    if (!ms || n < 0 || n > 5) { acb_set_error("bad argument"); return ACB_EINVAL; }
    for (int i = 0; i < n; i++) ms[i] = g_ll_ms[i];
    return ACB_OK;
}

static bool select_kind_ok(int kind) {
    if (kind == ACB_SELECT_LONGEST || kind == ACB_SELECT_FIRST) return true;
    acb_set_error("selection kind %d is neither ACB_SELECT_LONGEST nor ACB_SELECT_FIRST", kind);
    return false;
}

/* acb_leftmost_longest_device / acb_leftmost_first_device: the kind picks the sort order of step 1 (the candidate of a
 * (hay, start) run is its first record), nothing else */
static int leftmost_select(acb_table *tb, int kind, const acb_match *d_records, int64_t n, int64_t n_hay, int64_t max_hay_letters,
                           acb_match *d_out, int64_t cap, int64_t *d_count, cudaStream_t s) {
    if (!tb || n < 0 || (n && !d_records) || n_hay < 0 || max_hay_letters < 0 || cap < 0 || (cap > 0 && !d_out) || !d_count) {
        acb_set_error("bad argument");
        return ACB_EINVAL;
    }
    if (!select_kind_ok(kind)) return ACB_EINVAL;
    if (n > 0x7fffffffLL) { acb_set_error("more than 2^31-1 records to select from"); return ACB_ERANGE; }
    for (float &v : g_ll_ms) v = 0.f;
    if (n == 0) return ACB_OK;
    CUDA_TRY(cudaSetDevice(tb->device));
    const SortKey k = sort_key(tb, n_hay, max_hay_letters, kind);
    const int ni = (int)n;
    const long long n_tiles = (n + kLlTile - 1) / kLlTile;
    size_t t_sort = 0, t_sel = 0, t_scan = 0;
    CUDA_TRY(cub::DeviceRadixSort::SortPairs(nullptr, t_sort, (const unsigned long long *)nullptr, (unsigned long long *)nullptr,
                                             (const acb_match *)nullptr, (acb_match *)nullptr, ni, 0, 64, s));
    CUDA_TRY(cub::DeviceSelect::Flagged(nullptr, t_sel, (const acb_match *)nullptr, (const uint8_t *)nullptr, (acb_match *)nullptr,
                                        (unsigned long long *)nullptr, ni, s));
    CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, t_scan, (int32_t *)nullptr, (int32_t *)nullptr, ni, s));
    const size_t temp = std::max(t_sort, std::max(t_sel, t_scan));
    const size_t N = (size_t)n;
    const size_t need = 8 * 256 + 2 * N * sizeof(unsigned long long) + 2 * N * sizeof(acb_match) + N + 2 * N * sizeof(int32_t) +
                        (size_t)n_tiles * sizeof(unsigned long long) + temp;
    int rc;
    if ((rc = scratch_take(tb->l_buf, need, s))) return rc;
    if (!tb->l_ctr) CUDA_TRY(cudaMalloc(reinterpret_cast<void **>(&tb->l_ctr), 4 * sizeof(unsigned long long)));
    char *p = static_cast<char *>(tb->l_buf.buf);
    unsigned long long *k0 = carve<unsigned long long>(p, N), *k1 = carve<unsigned long long>(p, N);
    acb_match *ra = carve<acb_match>(p, N), *rb = carve<acb_match>(p, N);
    uint8_t *flag = carve<uint8_t>(p, N);
    int32_t *nxt = carve<int32_t>(p, N), *pos = carve<int32_t>(p, N);
    unsigned long long *status = carve<unsigned long long>(p, (size_t)n_tiles);
    void *tmp = carve<char>(p, temp);
    size_t tb_temp = temp;
    const unsigned grid = blocks(tb, n);
    if ((rc = timing_mark(&tb->l_ev[0], s))) return rc;
    /* 1. sort by start, then longest first or smallest key id first */
    rc = kind == ACB_SELECT_FIRST
             ? sort_records<kKeyFirst, kKeyFirstLow>(tb, k, d_records, rb, ra, n, k0, k1, tmp, temp, s, "leftmost sort key")
             : sort_records<kKeyStart, kKeyStartLow>(tb, k, d_records, rb, ra, n, k0, k1, tmp, temp, s, "leftmost sort key");
    if (rc || (rc = timing_mark(&tb->l_ev[1], s))) return rc;
    /* 2. candidates: the longest (first) match at every (hay, start) */
    acb_ll_cand_kernel<<<grid, 256, 0, s>>>(ra, n, tb->d_keylen, flag);
    if ((rc = launched("leftmost candidates"))) return rc;
    tb_temp = temp;
    CUDA_TRY(cub::DeviceSelect::Flagged(tmp, tb_temp, ra, flag, rb, tb->l_ctr, ni, s));
    if ((rc = timing_mark(&tb->l_ev[2], s))) return rc;
    /* 3. successors */
    acb_ll_next_kernel<<<grid, 256, 0, s>>>(rb, tb->l_ctr, tb->d_keylen, nxt);
    if ((rc = launched("leftmost successors")) || (rc = timing_mark(&tb->l_ev[3], s))) return rc;
    /* 4. chain marking */
    CUDA_TRY(cudaMemsetAsync(status, 0, (size_t)n_tiles * sizeof(unsigned long long), s));
    CUDA_TRY(cudaMemsetAsync(pos, 0, N * sizeof(int32_t), s));
    CUDA_TRY(cudaMemsetAsync(tb->l_ctr + 1, 0, sizeof(unsigned long long), s));
    acb_ll_chain_kernel<<<(unsigned)n_tiles, kLlThreads, 0, s>>>(rb, tb->l_ctr, nxt, std::max(k.max_len, 1), tb->l_ctr + 1, status, flag, pos);
    if ((rc = launched("leftmost chain")) || (rc = timing_mark(&tb->l_ev[4], s))) return rc;
    /* 5. emit */
    if ((rc = emit_flagged(tb, rb, tb->l_ctr, flag, pos, ni, tmp, temp, d_out, cap, d_count, s, "leftmost emit")) ||
        (rc = timing_mark(&tb->l_ev[5], s)) || (rc = scratch_done(&tb->l_buf.done, s)))
        return rc;
    for (int k = 0; k < 5; k++)
        if ((rc = timing_ms(tb->l_ev[k], tb->l_ev[k + 1], &g_ll_ms[k]))) return rc;
    return ACB_OK;
}

extern "C" int acb_leftmost_longest_device(acb_table *tb, const acb_match *d_records, int64_t n, int64_t n_hay,
                                           int64_t max_hay_letters, acb_match *d_out, int64_t cap, int64_t *d_count, void *stream) {
    DeviceRestore keep_device;
    return leftmost_select(tb, ACB_SELECT_LONGEST, d_records, n, n_hay, max_hay_letters, d_out, cap, d_count,
                           reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int acb_leftmost_first_device(acb_table *tb, const acb_match *d_records, int64_t n, int64_t n_hay,
                                         int64_t max_hay_letters, acb_match *d_out, int64_t cap, int64_t *d_count, void *stream) {
    DeviceRestore keep_device;
    return leftmost_select(tb, ACB_SELECT_FIRST, d_records, n, n_hay, max_hay_letters, d_out, cap, d_count,
                           reinterpret_cast<cudaStream_t>(stream));
}

/* ------------------------------------------------------------ whole-word filter */
/* A record is a whole-word match when neither the letter before its start nor the letter after its end is a word letter;
 * a haystack edge counts as a non-word letter, so a neighbour is never read from another haystack.  acb_ww_flag_kernel
 * flags every record (its key's length from the table, one or two neighbour letters, a bitmap lookup each); the kept
 * records are then compacted in order by the selection's emit step: exclusive sum of the flags, acb_ll_emit_kernel,
 * acb_ll_count_kernel. */
namespace {
thread_local float g_ww_ms = 0.f;                          /* kernel timing: flags to count */

/* a word set: letter v is a word letter iff v < n_bits and bit v is set */
struct WordBits {
    const uint32_t *bits;
    long long n_bits;

    /* for 1-byte letters, the set with its bitmap copied to s[8] in shared memory; every thread of the block calls it */
    template <int L>
    __device__ __forceinline__ WordBits shared(uint32_t *s) const {
        if (L != 1) return *this;
        if (threadIdx.x < 8) s[threadIdx.x] = (long long)threadIdx.x * 32 < n_bits ? bits[threadIdx.x] : 0u;
        __syncthreads();
        return {s, n_bits};
    }
    template <int L>
    __device__ __forceinline__ bool is_word(uint32_t v) const {
        if ((long long)v >= n_bits) return false;
        return ((L == 1 ? bits[v >> 5] : __ldg(bits + (v >> 5))) >> (v & 31) & 1u) != 0;
    }
};

struct WwArgs {
    const uint8_t *hay;
    const long long *off;                                  /* n_hay + 1 byte offsets, or nullptr: fixed stride (hay_start) */
    long long stride;
    const int32_t *key_len;
    WordBits words;
};

/* the letter at p, little-endian, at any alignment */
template <int L>
__device__ __forceinline__ uint32_t ww_letter(const uint8_t *p) {
    uint32_t v = __ldg(p);
    if (L >= 2) v |= (uint32_t)__ldg(p + 1) << 8;
    if (L == 4) v |= (uint32_t)__ldg(p + 2) << 16 | (uint32_t)__ldg(p + 3) << 24;
    return v;
}

/* flag[i] = pos[i] = record i is a whole-word match; *d_n = n (the emit step reads the count from the device) */
template <int L>
__global__ void __launch_bounds__(256) acb_ww_flag_kernel(const __grid_constant__ WwArgs a, const acb_match *rec, long long n,
                                                         uint8_t *flag, int32_t *pos, unsigned long long *d_n) {
    __shared__ uint32_t s_bits[8];
    const WordBits w = a.words.shared<L>(s_bits);
    const long long first = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (first == 0) *d_n = (unsigned long long)n;
    for (long long i = first; i < n; i += (long long)gridDim.x * blockDim.x) {
        const acb_match m = rec[i];
        const long long b0 = hay_start(a.off, a.stride, m.hay_id), letters = (hay_start(a.off, a.stride, m.hay_id + 1) - b0) / L;
        const long long end = m.end_index, start = end - __ldg(a.key_len + m.key_id) + 1;
        bool keep = start == 0 || !w.is_word<L>(ww_letter<L>(a.hay + b0 + (start - 1) * L));
        keep = keep && (end + 1 == letters || !w.is_word<L>(ww_letter<L>(a.hay + b0 + (end + 1) * L)));
        flag[i] = keep;
        pos[i] = keep;
    }
}
} // namespace

extern "C" int acb_last_words_ms(float *ms) {
    if (!ms) { acb_set_error("bad argument"); return ACB_EINVAL; }
    *ms = g_ww_ms;
    return ACB_OK;
}

/* a word bitmap of n_bits bits for the table's letters: at most one bit per letter value, bits given unless empty */
static int check_words(const acb_table *tb, const uint32_t *bits, int64_t n_bits) {
    const int64_t most = tb->L == 1 ? 256 : (tb->L == 2 ? 65536 : 0x110000);
    if (n_bits >= 0 && n_bits <= most && (bits || n_bits == 0)) return ACB_OK;
    acb_set_error("a word set of %d-byte letters has 0 .. %lld bits, and needs a bitmap unless it has none", tb->L, (long long)most);
    return ACB_EINVAL;
}

extern "C" int acb_word_filter_device(acb_table *tb, const uint8_t *d_hay, int64_t total_bytes, const int64_t *d_offsets, int64_t n_hay,
                                      int64_t stride_bytes, const acb_match *d_records, int64_t n, const uint32_t *d_bits, int64_t n_bits,
                                      acb_match *d_out, int64_t cap, int64_t *d_count, void *stream) {
    DeviceRestore keep_device;
    if (!tb || total_bytes < 0 || (total_bytes && !d_hay) || n_hay < 0 || n < 0 || (n && !d_records) || cap < 0 || (cap > 0 && !d_out) ||
        !d_count) {
        acb_set_error("bad argument");
        return ACB_EINVAL;
    }
    int rc;
    if ((rc = check_words(tb, d_bits, n_bits))) return rc;
    if (!d_offsets && (rc = check_stride(tb->L, total_bytes, n_hay, stride_bytes, 0))) return rc;
    if (n > 0x7fffffffLL) { acb_set_error("more than 2^31-1 records to filter"); return ACB_ERANGE; }
    g_ww_ms = 0.f;
    if (n == 0) return ACB_OK;
    CUDA_TRY(cudaSetDevice(tb->device));
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    const int ni = (int)n;
    const size_t N = (size_t)n;
    size_t temp = 0;
    CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, temp, (int32_t *)nullptr, (int32_t *)nullptr, ni, s));
    const size_t need = 3 * 256 + N + N * sizeof(int32_t) + sizeof(unsigned long long) + temp;
    if ((rc = scratch_take(tb->ww_buf, need, s))) return rc;
    char *p = static_cast<char *>(tb->ww_buf.buf);
    uint8_t *flag = carve<uint8_t>(p, N);
    int32_t *pos = carve<int32_t>(p, N);
    unsigned long long *d_n = carve<unsigned long long>(p, 1);
    void *tmp = carve<char>(p, temp);
    WwArgs a;
    a.hay = d_hay; a.off = reinterpret_cast<const long long *>(d_offsets); a.stride = stride_bytes; a.key_len = tb->d_keylen;
    a.words = {d_bits, n_bits};
    if ((rc = timing_mark(&tb->ww_ev[0], s))) return rc;
    with_width(tb->L, [&](auto w) { acb_ww_flag_kernel<decltype(w)::value><<<blocks(tb, n), 256, 0, s>>>(a, d_records, n, flag, pos, d_n); });
    if ((rc = launched("word flags")) || (rc = emit_flagged(tb, d_records, d_n, flag, pos, ni, tmp, temp, d_out, cap, d_count, s, "word filter emit")) ||
        (rc = timing_mark(&tb->ww_ev[1], s)) || (rc = scratch_done(&tb->ww_buf.done, s)))
        return rc;
    return timing_ms(tb->ww_ev[0], tb->ww_ev[1], &g_ww_ms);
}

/* ------------------------------------------------------------ alias expansion */
/* A folded table's scan reports each match under its group's representative, the lowest id of the keys that fold to the
 * same text.  The find_all routes then give every member of the group: record i becomes 1 + aliases(key_id) records,
 * the representative first and its aliases after it, ascending.  Count per record, exclusive sum, scatter. */
namespace {
struct XpArgs {
    const acb_match *rec;
    long long n;
    const int32_t *alias_ptr, *alias_ids;                  /* the table's alias CSR over n_rep ids (nullptr: no aliases) */
    int32_t n_rep;
};

__device__ __forceinline__ int32_t xp_aliases(const XpArgs &a, int32_t k, int32_t *first) {
    if (!a.alias_ptr || k < 0 || k >= a.n_rep) { *first = 0; return 0; }
    *first = __ldg(a.alias_ptr + k);
    return __ldg(a.alias_ptr + k + 1) - *first;
}

/* pos[i] = the records record i becomes; pos[n] = 0 (the exclusive sum then leaves the total there) */
__global__ void acb_xp_count_kernel(const __grid_constant__ XpArgs a, long long *pos) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i <= a.n; i += (long long)gridDim.x * blockDim.x) {
        int32_t first;
        pos[i] = i < a.n ? 1 + xp_aliases(a, a.rec[i].key_id, &first) : 0;
    }
}

/* the expanded records at out[pos[i] ..], those at or past cap not stored; *count = pos[n], the total */
__global__ void acb_xp_scatter_kernel(const __grid_constant__ XpArgs a, const long long *pos, acb_match *out, long long cap,
                                      long long *count) {
    const long long first_i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (first_i == 0) *count = pos[a.n];
    for (long long i = first_i; i < a.n; i += (long long)gridDim.x * blockDim.x) {
        acb_match m = a.rec[i];
        long long o = pos[i];
        int32_t first;
        const int32_t k = xp_aliases(a, m.key_id, &first);
        if (o < cap) out[o] = m;
        for (int32_t j = 0; j < k && ++o < cap; j++) {
            m.key_id = __ldg(a.alias_ids + first + j);
            out[o] = m;
        }
    }
}
} // namespace

extern "C" int acb_expand_aliases_device(acb_table *tb, const acb_match *d_in, int64_t n, acb_match *d_out, int64_t cap,
                                         int64_t *d_count, void *stream) {
    DeviceRestore keep_device;
    if (!tb || n < 0 || (n && !d_in) || cap < 0 || (cap > 0 && !d_out) || !d_count) { acb_set_error("bad argument"); return ACB_EINVAL; }
    if (!tb->fold) { acb_set_error("alias expansion needs a case-folded table (acb_table_upload_folded)"); return ACB_EINVAL; }
    /* the exclusive sum runs over n + 1 counts in an int */
    if (n >= 0x7fffffffLL) { acb_set_error("more than 2^31-2 records to expand"); return ACB_ERANGE; }
    g_fold_ms[1] = 0.f;
    CUDA_TRY(cudaSetDevice(tb->device));
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    if (n == 0) {
        CUDA_TRY(cudaMemsetAsync(d_count, 0, sizeof(int64_t), s));
        return ACB_OK;
    }
    const size_t N = (size_t)n + 1;
    size_t temp = 0;
    CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, temp, (long long *)nullptr, (long long *)nullptr, (int)N, s));
    int rc;
    if ((rc = scratch_take(tb->x_buf, 2 * 256 + N * sizeof(long long) + temp, s))) return rc;
    char *p = static_cast<char *>(tb->x_buf.buf);
    long long *pos = carve<long long>(p, N);
    void *tmp = carve<char>(p, temp);
    const XpArgs a{d_in, (long long)n, tb->d_alias_ptr, tb->d_alias_ids, tb->n_rep};
    if ((rc = timing_mark(&tb->f_ev[2], s))) return rc;
    acb_xp_count_kernel<<<blocks(tb, n + 1), 256, 0, s>>>(a, pos);
    if ((rc = launched("alias count"))) return rc;
    CUDA_TRY(cub::DeviceScan::ExclusiveSum(tmp, temp, pos, pos, (int)N, s));
    acb_xp_scatter_kernel<<<blocks(tb, n), 256, 0, s>>>(a, pos, d_out, cap, reinterpret_cast<long long *>(d_count));
    if ((rc = launched("alias scatter")) || (rc = timing_mark(&tb->f_ev[3], s)) || (rc = scratch_done(&tb->x_buf.done, s))) return rc;
    return timing_ms(tb->f_ev[2], tb->f_ev[3], &g_fold_ms[1]);
}

/* The host find_all routes on a table with aliases: the n records at *rec expanded into tb->x_out, grown to fit; then
 * *rec, *n and tb->w_count describe the expanded list.  Nothing without aliases.  On tb->stream, left synchronised. */
static int expand_host(acb_table *tb, acb_match **rec, unsigned long long *n) {
    if (!tb->n_alias || *n == 0) return ACB_OK;
    cudaStream_t s = tb->stream;
    int rc = ensure(&tb->x_out, &tb->x_out_cap, (size_t)*n);
    for (; rc == ACB_OK;) {
        if ((rc = acb_expand_aliases_device(tb, *rec, (int64_t)*n, tb->x_out, (int64_t)tb->x_out_cap, reinterpret_cast<int64_t *>(tb->w_count), s)))
            return rc;
        CUDA_TRY(cudaMemcpyAsync(tb->h_count, tb->w_count, sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
        CUDA_TRY(cudaStreamSynchronize(s));
        if (*tb->h_count <= tb->x_out_cap) break;
        rc = ensure(&tb->x_out, &tb->x_out_cap, (size_t)*tb->h_count);
    }
    if (rc != ACB_OK) return rc;
    *rec = tb->x_out;
    *n = *tb->h_count;
    return ACB_OK;
}

/* The word set of a host route that filters (acb_*_words): a host bitmap */
struct WordSet {
    const uint32_t *bits;
    int64_t n_bits;
};

/* The host routes' first step: the batch to tb->w_hay (and offsets to tb->w_off, *d_off), and its full match list into
 * tb->w_out, grown until it fits; *full is its length.  With a word set, the whole-word records of that list go on to
 * tb->ww_out and *full is their number.  *rec is the list the route goes on with, its length also in tb->w_count.  On
 * tb->stream, which it leaves synchronised. */
static int upload_and_scan_full(acb_table *tb, const uint8_t *hay, int64_t total_bytes, const int64_t *offsets, int64_t n_hay,
                                int64_t stride_bytes, int algo, const WordSet *ws, const int64_t **d_off, unsigned long long *full,
                                acb_match **rec) {
    int rc;
    if ((rc = upload_batch(tb, hay, total_bytes, offsets, n_hay, d_off)) ||
        (rc = ensure(&tb->w_out, &tb->w_out_cap, (size_t)std::max<int64_t>(2 * n_hay, 4096))))
        return rc;
    if (!tb->l_ctr) CUDA_TRY(cudaMalloc(reinterpret_cast<void **>(&tb->l_ctr), 4 * sizeof(unsigned long long)));
    cudaStream_t s = tb->stream;
    for (;;) {                                             /* the full list: an intermediate, in a buffer grown to fit */
        CUDA_TRY(cudaMemsetAsync(tb->w_count, 0, sizeof(unsigned long long), s));
        if ((rc = acb_scan_device(tb, tb->w_hay, total_bytes, *d_off, n_hay, stride_bytes, tb->w_out, (int64_t)tb->w_out_cap,
                                  reinterpret_cast<int64_t *>(tb->w_count), s, algo)))
            return rc;
        CUDA_TRY(cudaMemcpyAsync(tb->h_count, tb->w_count, sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
        CUDA_TRY(cudaStreamSynchronize(s));
        *full = *tb->h_count;
        if (*full <= tb->w_out_cap) break;
        if ((rc = ensure(&tb->w_out, &tb->w_out_cap, (size_t)*full))) return rc;
    }
    *rec = tb->w_out;
    if (!ws || *full == 0) return ACB_OK;
    const size_t words = ((size_t)ws->n_bits + 31) / 32;
    if ((rc = ensure(&tb->ww_bits, &tb->ww_bits_cap, std::max<size_t>(words, 1))) || (rc = ensure(&tb->ww_out, &tb->ww_out_cap, (size_t)*full)))
        return rc;
    if (words) CUDA_TRY(cudaMemcpyAsync(tb->ww_bits, ws->bits, words * sizeof(uint32_t), cudaMemcpyHostToDevice, s));
    CUDA_TRY(cudaMemsetAsync(tb->w_count, 0, sizeof(unsigned long long), s));
    if ((rc = acb_word_filter_device(tb, tb->w_hay, total_bytes, *d_off, n_hay, stride_bytes, tb->w_out, (int64_t)*full, tb->ww_bits,
                                     ws->n_bits, tb->ww_out, (int64_t)*full, reinterpret_cast<int64_t *>(tb->w_count), s)))
        return rc;
    CUDA_TRY(cudaMemcpyAsync(tb->h_count, tb->w_count, sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    *full = *tb->h_count;
    *rec = tb->ww_out;
    return ACB_OK;
}

/* the argument checks of the host routes that filter: the word set, and offsets, which the filter reads unchecked */
static int check_words_route(const acb_table *tb, const uint32_t *bits, int64_t n_bits, const int64_t *offsets, int64_t n_hay,
                             int64_t total_bytes) {
    int rc = check_words(tb, bits, n_bits);
    if (rc == ACB_OK && offsets) rc = check_offsets(tb->L, offsets, n_hay, total_bytes);
    return rc;
}

/* acb_scan_host_words, and without a word set (ws == nullptr) acb_scan_host on a table with aliases: the full list, its
 * whole-word records, expanded (expand_host), sorted and copied back */
static int scan_host_full(acb_table *tb, const uint8_t *hay, int64_t total_bytes, const int64_t *offsets, int64_t n_hay,
                          int64_t stride_bytes, const WordSet *ws, acb_match *out, int64_t cap, int64_t *n_found, int algo, int sort) {
    if (!tb || !n_found || total_bytes < 0 || n_hay < 0 || cap < 0 || (total_bytes && !hay)) { acb_set_error("bad argument"); return ACB_EINVAL; }
    *n_found = 0;
    if (algo != ACB_ALGO_AUTO && algo != ACB_ALGO_FILTER && algo != ACB_ALGO_DFA) { acb_set_error("a whole-word scan takes ACB_ALGO_AUTO, _FILTER or _DFA"); return ACB_EINVAL; }
    if (n_hay > 0x7fffffffLL) { acb_set_error("more than 2^31-1 haystacks in one batch"); return ACB_ERANGE; }
    int rc;
    if (ws && (rc = check_words_route(tb, ws->bits, ws->n_bits, offsets, n_hay, total_bytes))) return rc;
    if (!ws && offsets && (rc = check_offsets(tb->L, offsets, n_hay, total_bytes))) return rc;
    if (!offsets && (rc = check_stride(tb->L, total_bytes, n_hay, stride_bytes, 1))) return rc;
    tb->h_out_n = 0;
    if (total_bytes == 0 || n_hay == 0) return ACB_OK;
    const int64_t *d_off = nullptr;
    unsigned long long full = 0;
    acb_match *rec = nullptr;
    if ((rc = upload_and_scan_full(tb, hay, total_bytes, offsets, n_hay, stride_bytes, algo, ws, &d_off, &full, &rec)) ||
        (rc = expand_host(tb, &rec, &full)))
        return rc;
    return read_back(tb, tb->w_count, rec, cap, sort, n_hay, (offsets ? total_bytes : stride_bytes) / tb->L, out, n_found, tb->stream);
}

extern "C" int acb_scan_host_words(acb_table *tb, const uint8_t *hay, int64_t total_bytes, const int64_t *offsets, int64_t n_hay,
                                   int64_t stride_bytes, const uint32_t *bits, int64_t n_bits, acb_match *out, int64_t cap,
                                   int64_t *n_found, int algo, int sort) {
    DeviceRestore keep_device;
    const WordSet ws{bits, n_bits};
    return scan_host_full(tb, hay, total_bytes, offsets, n_hay, stride_bytes, &ws, out, cap, n_found, algo, sort);
}

static int scan_host_leftmost(acb_table *tb, const uint8_t *hay, int64_t total_bytes, const int64_t *offsets, int64_t n_hay,
                              int64_t stride_bytes, const WordSet *ws, acb_match *out, int64_t cap, int64_t *n_found, int algo,
                              int kind = ACB_SELECT_LONGEST) {
    if (!tb || !n_found || total_bytes < 0 || n_hay < 0 || cap < 0 || (total_bytes && !hay)) { acb_set_error("bad argument"); return ACB_EINVAL; }
    *n_found = 0;
    if (!select_kind_ok(kind)) return ACB_EINVAL;
    if (algo != ACB_ALGO_AUTO && algo != ACB_ALGO_FILTER && algo != ACB_ALGO_DFA) { acb_set_error("leftmost-longest takes ACB_ALGO_AUTO, _FILTER or _DFA"); return ACB_EINVAL; }
    if (n_hay > 0x7fffffffLL) { acb_set_error("more than 2^31-1 haystacks in one batch"); return ACB_ERANGE; }
    int rc;
    if (ws && (rc = check_words_route(tb, ws->bits, ws->n_bits, offsets, n_hay, total_bytes))) return rc;
    if (!offsets && (rc = check_stride(tb->L, total_bytes, n_hay, stride_bytes, 1))) return rc;
    tb->h_out_n = 0;
    if (total_bytes == 0 || n_hay == 0) return ACB_OK;
    const int64_t *d_off = nullptr;
    unsigned long long full = 0;
    acb_match *rec = nullptr;
    if ((rc = upload_and_scan_full(tb, hay, total_bytes, offsets, n_hay, stride_bytes, algo, ws, &d_off, &full, &rec))) return rc;
    cudaStream_t s = tb->stream;
    if (full == 0) return ACB_OK;
    const int64_t kept_cap = std::min<int64_t>(cap, (int64_t)full);
    if ((rc = ensure(&tb->l_out, &tb->l_out_cap, (size_t)std::max<int64_t>(kept_cap, 1)))) return rc;
    unsigned long long *d_n = tb->l_ctr + 2;
    CUDA_TRY(cudaMemsetAsync(d_n, 0, sizeof(unsigned long long), s));
    if ((rc = leftmost_select(tb, kind, rec, (int64_t)full, n_hay, (offsets ? total_bytes : stride_bytes) / tb->L, tb->l_out, kept_cap,
                              reinterpret_cast<int64_t *>(d_n), s)))
        return rc;
    return read_back(tb, d_n, tb->l_out, cap, 0, n_hay, 0, out, n_found, s);
}

extern "C" int acb_scan_host_leftmost(acb_table *tb, const uint8_t *hay, int64_t total_bytes, const int64_t *offsets, int64_t n_hay,
                                      int64_t stride_bytes, acb_match *out, int64_t cap, int64_t *n_found, int algo) {
    DeviceRestore keep_device;
    return scan_host_leftmost(tb, hay, total_bytes, offsets, n_hay, stride_bytes, nullptr, out, cap, n_found, algo);
}

extern "C" int acb_scan_host_leftmost_words(acb_table *tb, const uint8_t *hay, int64_t total_bytes, const int64_t *offsets, int64_t n_hay,
                                            int64_t stride_bytes, const uint32_t *bits, int64_t n_bits, acb_match *out, int64_t cap,
                                            int64_t *n_found, int algo) {
    DeviceRestore keep_device;
    const WordSet ws{bits, n_bits};
    return scan_host_leftmost(tb, hay, total_bytes, offsets, n_hay, stride_bytes, &ws, out, cap, n_found, algo);
}

extern "C" int acb_scan_host_leftmost_kind(acb_table *tb, int kind, const uint8_t *hay, int64_t total_bytes, const int64_t *offsets,
                                           int64_t n_hay, int64_t stride_bytes, const uint32_t *bits, int64_t n_bits, acb_match *out,
                                           int64_t cap, int64_t *n_found, int algo) {
    DeviceRestore keep_device;
    const WordSet ws{bits, n_bits};
    const bool words = n_bits >= 0 || bits;                 /* n_bits < 0 without a bitmap: no word filter */
    return scan_host_leftmost(tb, hay, total_bytes, offsets, n_hay, stride_bytes, words ? &ws : nullptr, out, cap, n_found, algo, kind);
}

/* ------------------------------------------------------------ leftmost-longest replacement */
/* The chosen records of a batch (acb_leftmost_longest_device's order) rewrite it: the letters of every chosen match
 * become the key's replacement, every other letter is copied.  Two passes:
 *  - offsets: D = exclusive scan of (rep_len - key_len * L) over the records.  Record i starts at input byte S_i (batch
 *    coordinates) and its replacement at output byte P_i = S_i + D[i]; it ends at E_i = P_i + rep_len, where the input
 *    resumes at IE_i = S_i + key_len * L.  Haystack h starts at out_off[h] = in_off[h] + D[lo_h], lo_h its first record
 *    (a binary search on hay_id); out_off[n_hay] is the total.
 *  - write: the output is cut into tiles of kRpTile bytes, whatever the haystacks.  ts[t] = the last record with
 *    P <= t * kRpTile (a binary search per tile), so the records that touch tile t are ts[t] .. ts[t+1]; a block stages
 *    them in shared memory (when they fit) and each thread writes one 16-byte chunk.  For an output byte o, k = the last
 *    record with P_k <= o: o < E_k is replacement byte RS_k + o - P_k, else o is copied from input byte IE_k + o - E_k
 *    (o itself before the first record).  A chunk inside one copy run or one replacement is one aligned 16-byte store
 *    of two aligned 16-byte loads merged by funnel shifts; only chunks that straddle a boundary go byte by byte. */
struct acb_replacer {
    int device = 0;
    int32_t L = 1;
    int64_t n_ids = 0;
    int kind = ACB_SELECT_LONGEST;                           /* the selection whose matches it rewrites */
    uint8_t *d_rep = nullptr;                                /* replacement bytes, 32 bytes of padding behind */
    long long *d_rep_off = nullptr;                          /* n_ids + 1 byte offsets */
};

namespace {
constexpr int kRpThreads = 256;
constexpr int kRpTile = kRpThreads * 16;                   /* output bytes per tile: one 16-byte chunk per thread */
constexpr int kRpStage = 512;                              /* records a tile stages in shared memory */
thread_local float g_rp_ms[2] = {};                        /* kernel timing: offsets pass, write pass */

struct RpArgs {
    const acb_match *chosen; const unsigned long long *n_chosen; long long cap;   /* records: min(*n_chosen, cap) */
    const int32_t *key_len; const long long *rep_off; const uint8_t *rep; int L;
    const uint8_t *hay; const long long *in_off; long long stride, n_hay, total_bytes;
    long long *D, *P, *E, *IE, *RS;                        /* D[cap + 1]; the others per record */
    long long *ts; long long out_cap;
    long long *out_off, *total; uint8_t *out;
};

__device__ __forceinline__ long long rp_n(const RpArgs &a) { return min((long long)*a.n_chosen, a.cap); }

/* D[i] = rep_len - key_len * L of record i, 0 for i in [n, cap] (the exclusive scan then leaves the sum in D[cap]) */
__global__ void acb_rp_delta_kernel(const __grid_constant__ RpArgs a) {
    const long long n = rp_n(a);
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i <= a.cap; i += (long long)gridDim.x * blockDim.x) {
        long long d = 0;
        if (i < n) {
            const int k = a.chosen[i].key_id;
            d = a.rep_off[k + 1] - a.rep_off[k] - (long long)__ldg(a.key_len + k) * a.L;
        }
        a.D[i] = d;
    }
}

__global__ void acb_rp_records_kernel(const __grid_constant__ RpArgs a) {
    const long long n = rp_n(a);
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const acb_match m = a.chosen[i];
        const long long len = __ldg(a.key_len + m.key_id);
        const long long s = hay_start(a.in_off, a.stride, m.hay_id) + ((long long)m.end_index - len + 1) * a.L;
        const long long p = s + a.D[i], rs = a.rep_off[m.key_id];
        a.P[i] = p;
        a.E[i] = p + a.rep_off[m.key_id + 1] - rs;
        a.IE[i] = s + len * a.L;
        a.RS[i] = rs;
    }
}

/* out_off[h] = in_off[h] + D[first record of a haystack >= h], for h in [0, n_hay]; the last one is the total */
__global__ void acb_rp_offsets_kernel(const __grid_constant__ RpArgs a) {
    const long long n = rp_n(a);
    for (long long h = (long long)blockIdx.x * blockDim.x + threadIdx.x; h <= a.n_hay; h += (long long)gridDim.x * blockDim.x) {
        long long lo = 0, hi = n;
        while (lo < hi) {
            const long long mid = (lo + hi) >> 1;
            if ((long long)a.chosen[mid].hay_id < h) lo = mid + 1; else hi = mid;
        }
        const long long o = (h == a.n_hay ? a.total_bytes : hay_start(a.in_off, a.stride, h)) + a.D[lo];
        a.out_off[h] = o;
        if (h == a.n_hay) *a.total = o;
    }
}

/* last j in [lo, hi] with P[j - base] <= o, or lo - 1 */
__device__ __forceinline__ long long rp_find(const long long *P, long long base, long long lo, long long hi, long long o) {
    while (lo <= hi) {
        const long long mid = (lo + hi) >> 1;
        if (P[mid - base] <= o) lo = mid + 1; else hi = mid - 1;
    }
    return hi;
}

/* ts[t] = the last record with P <= t * kRpTile, for t in [0, n_tiles]; nothing when the output does not fit */
__global__ void acb_rp_tiles_kernel(const __grid_constant__ RpArgs a) {
    const long long total = *a.total;
    if (total > a.out_cap) return;
    const long long n = rp_n(a), n_tiles = (total + kRpTile - 1) / kRpTile;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t <= n_tiles; t += (long long)gridDim.x * blockDim.x)
        a.ts[t] = rp_find(a.P, 0, 0, n - 1, t * kRpTile);
}

/* 16 bytes from p + x, p 16-byte aligned: two aligned loads (one when x is aligned) merged by funnel shifts.  The
 * second block holds byte x + 15 - (x & 15) + 16 > x + 15 only when x is not aligned, so it always holds a byte of [x, x + 16) */
__device__ __forceinline__ uint4 rp_load16(const uint8_t *p, long long x) {
    const uint4 v0 = __ldg(reinterpret_cast<const uint4 *>(p + (x & ~15LL)));
    const int off = (int)(x & 15);
    if (off == 0) return v0;
    const uint4 v1 = __ldg(reinterpret_cast<const uint4 *>(p + (x & ~15LL) + 16));
    const uint32_t w[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
    const int q = off >> 2, r = (off & 3) * 8;
    uint32_t s[5];
#pragma unroll
    for (int j = 0; j < 5; j++) s[j] = q == 0 ? w[j] : q == 1 ? w[j + 1] : q == 2 ? w[j + 2] : (j + 3 < 8 ? w[j + 3] : 0u);
    return make_uint4(__funnelshift_r(s[0], s[1], r), __funnelshift_r(s[1], s[2], r), __funnelshift_r(s[2], s[3], r),
                      __funnelshift_r(s[3], s[4], r));
}

__global__ void __launch_bounds__(kRpThreads) acb_rp_write_kernel(const __grid_constant__ RpArgs a) {
    __shared__ long long sP[kRpStage], sE[kRpStage], sIE[kRpStage], sRS[kRpStage];
    const long long total = *a.total;
    if (total > a.out_cap) return;
    const long long n_tiles = (total + kRpTile - 1) / kRpTile;
    for (long long t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        const long long lo = max(a.ts[t], 0LL), hi = a.ts[t + 1], m = hi - lo + 1;
        const bool staged = m > 0 && m <= kRpStage;
        __syncthreads();                                   /* the previous tile's readers are done */
        if (staged) {
            for (int j = threadIdx.x; j < m; j += kRpThreads) {
                sP[j] = a.P[lo + j]; sE[j] = a.E[lo + j]; sIE[j] = a.IE[lo + j]; sRS[j] = a.RS[lo + j];
            }
        }
        __syncthreads();
        const long long *P = staged ? sP : a.P, *E = staged ? sE : a.E, *IE = staged ? sIE : a.IE, *RS = staged ? sRS : a.RS;
        const long long base = staged ? lo : 0;
        const long long c = t * kRpTile + (long long)threadIdx.x * 16;
        if (c >= total) continue;
        long long k = rp_find(P, base, lo, hi, c);
        const bool in_rep = k >= lo && c < E[k - base];
        if (in_rep && c + 16 <= E[k - base]) {
            *reinterpret_cast<uint4 *>(a.out + c) = rp_load16(a.rep, RS[k - base] + (c - P[k - base]));
            continue;
        }
        if (!in_rep && c + 16 <= total && (k == hi || c + 16 <= P[k + 1 - base])) {
            *reinterpret_cast<uint4 *>(a.out + c) = rp_load16(a.hay, k >= lo ? IE[k - base] + (c - E[k - base]) : c);
            continue;
        }
        uint32_t w[4] = {0u, 0u, 0u, 0u};                 /* a chunk across a boundary: byte by byte */
#pragma unroll
        for (int j = 0; j < 16; j++) {
            const long long o = c + j;
            if (o < total) {
                k = rp_find(P, base, max(k, lo), hi, o);
                uint32_t b;
                if (k >= lo && o < E[k - base]) b = __ldg(a.rep + RS[k - base] + (o - P[k - base]));
                else b = __ldg(a.hay + (k >= lo ? IE[k - base] + (o - E[k - base]) : o));
                w[j >> 2] |= b << (8 * (j & 3));
            }
        }
        if (c + 16 <= total) {
            *reinterpret_cast<uint4 *>(a.out + c) = make_uint4(w[0], w[1], w[2], w[3]);
        } else {
#pragma unroll
            for (int j = 0; j < 16; j++)
                if (c + j < total) a.out[c + j] = (uint8_t)(w[j >> 2] >> (8 * (j & 3)));
        }
    }
}
} // namespace

static int rp_fits(const acb_replacer *r, const acb_table *tb) {
    if (r->device != tb->device || r->L != tb->L || r->n_ids < tb->n_keys) {
        acb_set_error("replacer made for device %d, %d-byte letters and %lld key ids; table: device %d, %d-byte letters, %d key ids",
                      r->device, r->L, (long long)r->n_ids, tb->device, tb->L, tb->n_keys);
        return ACB_EINVAL;
    }
    return ACB_OK;
}

extern "C" int acb_replacer_new_kind(const acb_table *tb, int kind, const uint8_t *rep, int64_t rep_bytes, const int64_t *rep_offsets,
                                     int64_t n_ids, acb_replacer **out) {
    DeviceRestore keep_device;
    if (!tb || !out || rep_bytes < 0 || (rep_bytes && !rep) || !rep_offsets || n_ids < 0) { acb_set_error("bad argument"); return ACB_EINVAL; }
    *out = nullptr;
    if (!select_kind_ok(kind)) return ACB_EINVAL;
    if (tb->L != 1 && tb->L != 2 && tb->L != 4) { acb_set_error("not a table"); return ACB_EINVAL; }
    if (n_ids < tb->n_keys) { acb_set_error("%lld replacements for %d key ids", (long long)n_ids, tb->n_keys); return ACB_EINVAL; }
    int rc = check_offsets(tb->L, rep_offsets, n_ids, rep_bytes);
    if (rc != ACB_OK) return rc;
    CUDA_TRY(cudaSetDevice(tb->device));
    acb_replacer *r = new (std::nothrow) acb_replacer();
    if (!r) { acb_set_error("out of memory"); return ACB_ENOMEM; }
    r->device = tb->device; r->L = tb->L; r->n_ids = n_ids; r->kind = kind;
    cudaError_t e = cudaMalloc(reinterpret_cast<void **>(&r->d_rep), (size_t)rep_bytes + 32);
    if (e == cudaSuccess) e = cudaMalloc(reinterpret_cast<void **>(&r->d_rep_off), (size_t)(n_ids + 1) * sizeof(long long));
    if (e == cudaSuccess && rep_bytes) e = cudaMemcpy(r->d_rep, rep, (size_t)rep_bytes, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(r->d_rep_off, rep_offsets, (size_t)(n_ids + 1) * sizeof(long long), cudaMemcpyHostToDevice);
    if (e != cudaSuccess) {
        acb_set_error("CUDA error %s uploading the replacements: %s", cudaGetErrorName(e), cudaGetErrorString(e));
        acb_replacer_free(r);
        return ACB_ECUDA;
    }
    *out = r;
    return ACB_OK;
}

extern "C" int acb_replacer_new(const acb_table *tb, const uint8_t *rep, int64_t rep_bytes, const int64_t *rep_offsets,
                                int64_t n_ids, acb_replacer **out) {
    DeviceRestore keep_device;
    return acb_replacer_new_kind(tb, ACB_SELECT_LONGEST, rep, rep_bytes, rep_offsets, n_ids, out);
}

extern "C" void acb_replacer_free(acb_replacer *r) {
    DeviceRestore keep_device;
    if (!r) return;
    cudaSetDevice(r->device);
    cudaFree(r->d_rep);
    cudaFree(r->d_rep_off);
    delete r;
}

extern "C" int acb_last_replace_ms(float *ms, int32_t n) {
    if (!ms || n < 0 || n > 2) { acb_set_error("bad argument"); return ACB_EINVAL; }
    for (int i = 0; i < n; i++) ms[i] = g_rp_ms[i];
    return ACB_OK;
}

/* The offsets pass on s: a.out_off[0..n_hay] and *a.total.  Carves the per-record arrays from tb->r_buf. */
static int rp_offsets(acb_table *tb, RpArgs &a, cudaStream_t s) {
    const size_t C = (size_t)a.cap;
    size_t temp = 0;
    CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, temp, (long long *)nullptr, (long long *)nullptr, a.cap + 1, s));
    const size_t need = 6 * 256 + (C + 1) * 8 + 4 * C * 8 + temp;
    int rc;
    if ((rc = scratch_take(tb->r_buf, need, s))) return rc;
    char *p = static_cast<char *>(tb->r_buf.buf);
    a.D = carve<long long>(p, C + 1);
    a.P = carve<long long>(p, C);
    a.E = carve<long long>(p, C);
    a.IE = carve<long long>(p, C);
    a.RS = carve<long long>(p, C);
    void *tmp = carve<char>(p, temp);
    if ((rc = timing_mark(&tb->r_ev[0], s))) return rc;
    acb_rp_delta_kernel<<<blocks(tb, a.cap + 1), 256, 0, s>>>(a);
    if ((rc = launched("replacement delta"))) return rc;
    CUDA_TRY(cub::DeviceScan::ExclusiveSum(tmp, temp, a.D, a.D, a.cap + 1, s));
    if (a.cap) {
        acb_rp_records_kernel<<<blocks(tb, a.cap), 256, 0, s>>>(a);
        if ((rc = launched("replacement records"))) return rc;
    }
    acb_rp_offsets_kernel<<<blocks(tb, a.n_hay + 1), 256, 0, s>>>(a);
    if ((rc = launched("replacement offsets"))) return rc;
    return timing_mark(&tb->r_ev[1], s);
}

/* The write pass on s: a.out, when *a.total <= a.out_cap (checked on the device).  Then the scratch event and timing. */
static int rp_write(acb_table *tb, RpArgs &a, cudaStream_t s) {
    int rc;
    if ((rc = timing_mark(&tb->r_ev[2], s))) return rc;
    if (a.out_cap > 0) {
        const long long max_tiles = (a.out_cap + kRpTile - 1) / kRpTile;
        if (tb->r_ts_cap < (size_t)max_tiles + 1) {
            CUDA_TRY(cudaStreamSynchronize(s));
            if ((rc = ensure(&tb->r_ts, &tb->r_ts_cap, (size_t)max_tiles + 1))) return rc;
        }
        a.ts = tb->r_ts;
        acb_rp_tiles_kernel<<<blocks(tb, max_tiles + 1), 256, 0, s>>>(a);
        if ((rc = launched("replacement tiles"))) return rc;
        acb_rp_write_kernel<<<(unsigned)std::min<long long>(max_tiles, grid_sms(tb) * 8), kRpThreads, 0, s>>>(a);
        if ((rc = launched("replacement write"))) return rc;
    }
    if ((rc = timing_mark(&tb->r_ev[3], s)) || (rc = scratch_done(&tb->r_buf.done, s)) || (rc = timing_ms(tb->r_ev[0], tb->r_ev[1], &g_rp_ms[0])))
        return rc;
    return timing_ms(tb->r_ev[2], tb->r_ev[3], &g_rp_ms[1]);
}

static int rp_check(const acb_replacer *r, const acb_table *tb, int64_t total_bytes, int64_t n_hay, int64_t stride_bytes,
                    bool has_offsets, int64_t out_cap) {
    if (!r || !tb || total_bytes < 0 || n_hay < 0 || out_cap < 0) { acb_set_error("bad argument"); return ACB_EINVAL; }
    int rc = rp_fits(r, tb);
    if (rc) return rc;
    if (n_hay > 0x7fffffffLL) { acb_set_error("more than 2^31-1 haystacks in one batch"); return ACB_ERANGE; }
    return has_offsets ? ACB_OK : check_stride(tb->L, total_bytes, n_hay, stride_bytes, 0);
}

static void rp_args(RpArgs &a, const acb_replacer *r, const acb_table *tb, const uint8_t *d_hay, int64_t total_bytes,
                    const int64_t *d_offsets, int64_t n_hay, int64_t stride_bytes, const acb_match *d_chosen, int64_t chosen_cap,
                    const int64_t *d_n_chosen, int64_t *d_out_offsets, uint8_t *d_out, int64_t out_cap, int64_t *d_total) {
    a = RpArgs{};
    a.chosen = d_chosen; a.n_chosen = reinterpret_cast<const unsigned long long *>(d_n_chosen); a.cap = chosen_cap;
    a.key_len = tb->d_keylen; a.rep_off = r->d_rep_off; a.rep = r->d_rep; a.L = tb->L;
    a.hay = d_hay; a.in_off = reinterpret_cast<const long long *>(d_offsets); a.stride = stride_bytes; a.n_hay = n_hay;
    a.total_bytes = total_bytes; a.out_cap = out_cap;
    a.out_off = reinterpret_cast<long long *>(d_out_offsets); a.total = reinterpret_cast<long long *>(d_total); a.out = d_out;
}

extern "C" int acb_replace_device(acb_replacer *r, acb_table *tb, const uint8_t *d_hay, int64_t total_bytes, const int64_t *d_offsets,
                                  int64_t n_hay, int64_t stride_bytes, const acb_match *d_chosen, int64_t chosen_cap,
                                  const int64_t *d_n_chosen, int64_t *d_out_offsets, uint8_t *d_out, int64_t out_cap,
                                  int64_t *d_total, void *stream) {
    DeviceRestore keep_device;
    int rc = rp_check(r, tb, total_bytes, n_hay, stride_bytes, d_offsets != nullptr, out_cap);
    if (rc) return rc;
    if ((total_bytes && !d_hay) || chosen_cap < 0 || (chosen_cap && !d_chosen) || !d_n_chosen || !d_out_offsets || !d_total ||
        (out_cap && !d_out)) {
        acb_set_error("bad argument");
        return ACB_EINVAL;
    }
    if ((reinterpret_cast<uintptr_t>(d_hay) | reinterpret_cast<uintptr_t>(d_out)) & 15) {
        acb_set_error("d_hay and d_out must be 16-byte aligned");
        return ACB_EINVAL;
    }
    for (float &v : g_rp_ms) v = 0.f;
    CUDA_TRY(cudaSetDevice(tb->device));
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    RpArgs a;
    rp_args(a, r, tb, d_hay, total_bytes, d_offsets, n_hay, stride_bytes, d_chosen, chosen_cap, d_n_chosen, d_out_offsets, d_out,
            out_cap, d_total);
    if ((rc = rp_offsets(tb, a, s))) return rc;
    return rp_write(tb, a, s);
}

static int replace_host(acb_replacer *r, acb_table *tb, const uint8_t *hay, int64_t total_bytes, const int64_t *offsets, int64_t n_hay,
                        int64_t stride_bytes, const WordSet *ws, int algo, int64_t *out_offsets, uint8_t *out, int64_t out_cap, int64_t *total) {
    int rc = rp_check(r, tb, total_bytes, n_hay, stride_bytes, offsets != nullptr, out_cap);
    if (rc) return rc;
    if ((total_bytes && !hay) || !out_offsets || !total || (out_cap && !out)) { acb_set_error("bad argument"); return ACB_EINVAL; }
    if (algo != ACB_ALGO_AUTO && algo != ACB_ALGO_FILTER && algo != ACB_ALGO_DFA) { acb_set_error("replacement takes ACB_ALGO_AUTO, _FILTER or _DFA"); return ACB_EINVAL; }
    if (offsets && (rc = check_offsets(tb->L, offsets, n_hay, total_bytes))) return rc;
    if (ws && (rc = check_words(tb, ws->bits, ws->n_bits))) return rc;
    *total = 0;
    for (float &v : g_rp_ms) v = 0.f;
    if (n_hay == 0) { out_offsets[0] = 0; return ACB_OK; }
    const int64_t *d_off = nullptr;
    unsigned long long full = 0;
    acb_match *rec = nullptr;
    if (total_bytes && (rc = upload_and_scan_full(tb, hay, total_bytes, offsets, n_hay, stride_bytes, algo, ws, &d_off, &full, &rec))) return rc;
    if (!total_bytes) {                                     /* only empty haystacks: nothing to scan, nothing to write */
        for (int64_t i = 0; i <= n_hay; i++) out_offsets[i] = 0;
        return ACB_OK;
    }
    cudaStream_t s = tb->stream;
    if ((rc = ensure(&tb->r_off, &tb->r_off_cap, (size_t)n_hay + 2))) return rc;
    unsigned long long *d_n = tb->l_ctr + 2;
    CUDA_TRY(cudaMemsetAsync(d_n, 0, sizeof(unsigned long long), s));
    if (full && (rc = ensure(&tb->l_out, &tb->l_out_cap, (size_t)full))) return rc;
    if (full && (rc = leftmost_select(tb, r->kind, rec, (int64_t)full, n_hay, (offsets ? total_bytes : stride_bytes) / tb->L,
                                      tb->l_out, (int64_t)full, reinterpret_cast<int64_t *>(d_n), s)))
        return rc;
    RpArgs a;
    rp_args(a, r, tb, tb->w_hay, total_bytes, d_off, n_hay, stride_bytes, tb->l_out, (int64_t)full, reinterpret_cast<int64_t *>(d_n),
            reinterpret_cast<int64_t *>(tb->r_off), nullptr, 0, reinterpret_cast<int64_t *>(tb->r_off + n_hay + 1));
    if ((rc = rp_offsets(tb, a, s))) return rc;
    CUDA_TRY(cudaMemcpyAsync(out_offsets, tb->r_off, (size_t)(n_hay + 1) * sizeof(int64_t), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    *total = out_offsets[n_hay];
    if (*total > out_cap) {
        acb_set_error("replacement: room for %lld bytes, output %lld", (long long)out_cap, (long long)*total);
        return ACB_EOVERFLOW;
    }
    if ((rc = ensure(&tb->r_out, &tb->r_out_cap, (size_t)std::max<int64_t>(*total, 16)))) return rc;
    a.out = tb->r_out;
    a.out_cap = *total;
    if ((rc = rp_write(tb, a, s))) return rc;
    if (*total) CUDA_TRY(cudaMemcpyAsync(out, tb->r_out, (size_t)*total, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    return ACB_OK;
}

extern "C" int acb_replace_host(acb_replacer *r, acb_table *tb, const uint8_t *hay, int64_t total_bytes, const int64_t *offsets,
                                int64_t n_hay, int64_t stride_bytes, int algo, int64_t *out_offsets, uint8_t *out, int64_t out_cap,
                                int64_t *total) {
    DeviceRestore keep_device;
    return replace_host(r, tb, hay, total_bytes, offsets, n_hay, stride_bytes, nullptr, algo, out_offsets, out, out_cap, total);
}

extern "C" int acb_replace_host_words(acb_replacer *r, acb_table *tb, const uint8_t *hay, int64_t total_bytes, const int64_t *offsets,
                                      int64_t n_hay, int64_t stride_bytes, const uint32_t *bits, int64_t n_bits, int algo, int64_t *out_offsets,
                                      uint8_t *out, int64_t out_cap, int64_t *total) {
    DeviceRestore keep_device;
    const WordSet ws{bits, n_bits};
    return replace_host(r, tb, hay, total_bytes, offsets, n_hay, stride_bytes, &ws, algo, out_offsets, out, out_cap, total);
}

/* ------------------------------------------------------------ leftmost-longest stream batches */
/* A leftmost-longest stream batch keeps, per stream, X: the position up to which every match is decided and emitted,
 * and in its tail the pos - X <= T letters after it.  A feed:
 *  1. stages held || chunk per chunk (a length kernel, an exclusive scan, a tiled gather);
 *  2. scans the staged batch with acb_scan_device: from the root at X it finds exactly the matches that start at or
 *     after X, since the greedy chain has no match starting in [last chosen end + 1, X);
 *  3. keeps the records that start before the frontier F = pos_new - T (all of them on a final feed): they end before
 *     pos_new, so every match that can decide a choice among them is known;
 *  4. selects with acb_leftmost_longest_device;
 *  5. computes X_new = max(X, F, end of the last chosen record + 1) (pos_new on a final feed) and, for a replacing
 *     feed, rewrites the windows [X, X_new) with acb_replace_device;
 *  6. commits the new held letters, X and the position, only when everything fit the caller's buffers.
 * DESIGN section 4.13 gives the exactness argument. */
namespace {
constexpr int kSlTile = 4096;                              /* output bytes per block turn of the ragged gather */
constexpr int kSlHays = 512;                               /* haystack offsets a gather block keeps in shared memory */
constexpr int kSlLanes = 8;                                /* lanes per chunk of the commit's tail copy */
thread_local float g_sl_ms[6] = {};                        /* kernel timing: stage, scan, filter, selection, window, commit */

struct SlArgs {
    const int32_t *ids; long long n_streams;               /* chunk -> stream, as StreamsArgs */
    long long *pos, *hold; uint8_t *tail; int T, L;
    const uint8_t *chunks; const long long *off; long long stride;   /* the caller's chunks */
    long long n;                                           /* chunks */
    long long *soff;                                       /* staged byte offsets [n + 1] */
    uint8_t *stage;
    long long *last, *xn, *woff;                           /* per chunk: last chosen end (staged letters) or -1, new X
                                                              (staged letters), window byte offsets [n + 1] */
    int final;
};

__device__ __forceinline__ long long sl_stream(const SlArgs &a, long long h) {
    const long long s = a.ids ? (long long)__ldg(a.ids + h) : h;
    return (s >= 0 && s < a.n_streams) ? s : -1;
}

/* bytes of chunk h */
__device__ __forceinline__ long long sl_chunk_bytes(const SlArgs &a, long long h) {
    return hay_start(a.off, a.stride, h + 1) - hay_start(a.off, a.stride, h);
}

/* soff[h] = bytes of held || chunk h (soff[n] = 0), for the exclusive scan that makes them offsets */
__global__ void acb_sl_len_kernel(const __grid_constant__ SlArgs a) {
    for (long long h = (long long)blockIdx.x * blockDim.x + threadIdx.x; h <= a.n; h += (long long)gridDim.x * blockDim.x) {
        long long len = 0;
        if (h < a.n) {
            const long long s = sl_stream(a, h);
            len = sl_chunk_bytes(a, h) + (s < 0 ? 0 : a.hold[s] * a.L);
        }
        a.soff[h] = len;
    }
}

/* last j in [lo, hi] with o(j) <= x, o(lo) <= x */
template <class O>
__device__ __forceinline__ long long sl_find(const O &o, long long lo, long long hi, long long x) {
    while (lo < hi) {
        const long long mid = (lo + hi + 1) >> 1;
        if (o(mid) <= x) lo = mid; else hi = mid - 1;
    }
    return lo;
}

/* ts[t] = the haystack that holds output byte t * kSlTile (the last h with doff[h] <= it), one lane per tile */
__global__ void acb_sl_tiles_kernel(const long long *doff, long long n, long long total, long long *ts) {
    const long long n_tiles = (total + kSlTile - 1) / kSlTile;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < n_tiles; t += (long long)gridDim.x * blockDim.x)
        ts[t] = sl_find([&](long long j) { return doff[j]; }, 0, n - 1, t * kSlTile);
}

/* A ragged gather: output haystack h = [doff[h], doff[h+1]) is its first `head` bytes from the tail of its stream, then
 * the rest from a source haystack.  kStage: held || chunk (head = held letters, source = the caller's chunk); else the
 * window [X, X_new) (head = 0, source = the staged haystack).  Blocks take tiles of kSlTile output bytes, start at the
 * tile's first haystack ts[t] and keep the following offsets in shared memory; each thread writes one 16-byte chunk,
 * from two aligned 16-byte loads when it lies in one source run, else byte by byte. */
template <bool kStage>
__global__ void __launch_bounds__(256) acb_sl_gather_kernel(const __grid_constant__ SlArgs a, const long long *doff, const long long *ts,
                                                             uint8_t *dst, long long total) {
    __shared__ long long s_off[kSlHays + 1];
    const long long n_tiles = (total + kSlTile - 1) / kSlTile;
    const uint8_t *base = kStage ? a.chunks : a.stage;
    for (long long t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        const long long c0 = t * kSlTile, h0 = ts[t];
        const int nh = (int)min((long long)kSlHays, a.n - h0);
        __syncthreads();                                   /* the previous tile's readers are done */
        for (int j = threadIdx.x; j <= nh; j += blockDim.x) s_off[j] = doff[h0 + j];
        __syncthreads();
        const auto O = [&](long long j) { return j - h0 <= nh ? s_off[j - h0] : doff[j]; };
        const auto F = [&](long long from, long long x) {  /* within the shared offsets when x lies before their end */
            return sl_find(O, from, x < s_off[nh] ? h0 + nh - 1 : a.n - 1, x);
        };
        const long long c = c0 + (long long)threadIdx.x * 16;
        if (c >= total) continue;
        long long h = F(h0, c), lo = O(h), hi = O(h + 1), hd = 0;
        const uint8_t *tp = nullptr, *sp;                  /* the held letters; sp[o - lo] = source byte of output o */
        const auto enter = [&]() {
            if (kStage) {
                const long long s = sl_stream(a, h);
                hd = s < 0 ? 0 : a.hold[s] * a.L;
                tp = a.tail + (s < 0 ? 0 : s) * a.T * a.L;
            }
            sp = base + (kStage ? hay_start(a.off, a.stride, h) : a.soff[h]) - hd;
        };
        enter();
        if (c - lo >= hd && c + 16 <= hi) {
            *reinterpret_cast<uint4 *>(dst + c) = rp_load16(base, (sp - base) + (c - lo));
            continue;
        }
        uint32_t w[4] = {0u, 0u, 0u, 0u};
#pragma unroll
        for (int j = 0; j < 16; j++) {
            const long long o = c + j;
            if (o < total) {
                if (o >= hi) { h = F(h + 1, o); lo = O(h); hi = O(h + 1); enter(); }
                const long long rel = o - lo;
                const uint32_t b = rel < hd ? tp[rel] : sp[rel];
                w[j >> 2] |= b << (8 * (j & 3));
            }
        }
        if (c + 16 <= total) {
            *reinterpret_cast<uint4 *>(dst + c) = make_uint4(w[0], w[1], w[2], w[3]);
        } else {
#pragma unroll
            for (int j = 0; j < 16; j++)
                if (c + j < total) dst[c + j] = (uint8_t)(w[j >> 2] >> (8 * (j & 3)));
        }
    }
}

/* flag[i]: record i of the full list starts before its chunk's frontier (every record on a final feed) */
__global__ void acb_sl_flag_kernel(const __grid_constant__ SlArgs a, const acb_match *full, const unsigned long long *count,
                                   long long cap, const int32_t *key_len, uint8_t *flag) {
    const long long m = min((long long)*count, cap);
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < cap; i += (long long)gridDim.x * blockDim.x) {
        bool keep = false;
        if (i < m) {
            const acb_match r = full[i];
            const long long staged = (a.soff[r.hay_id + 1] - a.soff[r.hay_id]) / a.L;
            keep = a.final || (long long)r.end_index - __ldg(key_len + r.key_id) + 1 < staged - a.T;
        }
        flag[i] = keep;
    }
}

/* last[h] = end of chunk h's last chosen record (staged letters); rebase: end_index relative to the chunk */
__global__ void acb_sl_last_kernel(const __grid_constant__ SlArgs a, acb_match *rec, const unsigned long long *count, long long cap,
                                   int rebase) {
    const long long m = min((long long)*count, cap);
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += (long long)gridDim.x * blockDim.x) {
        const int32_t h = rec[i].hay_id, e = rec[i].end_index;
        if (i + 1 == m || rec[i + 1].hay_id != h) a.last[h] = e;
        if (rebase) {
            const long long s = sl_stream(a, h);
            rec[i].end_index = (int32_t)(e - (s < 0 ? 0 : a.hold[s]));
        }
    }
}

/* xn[h] = X_new - X in letters; woff[h] = its bytes (woff[n] = 0), for the exclusive scan that makes the window offsets */
__global__ void acb_sl_frontier_kernel(const __grid_constant__ SlArgs a) {
    for (long long h = (long long)blockIdx.x * blockDim.x + threadIdx.x; h <= a.n; h += (long long)gridDim.x * blockDim.x) {
        if (h == a.n) { a.woff[h] = 0; continue; }
        const long long staged = (a.soff[h + 1] - a.soff[h]) / a.L;
        const long long x = a.final ? staged : max(max(0LL, staged - a.T), a.last[h] + 1);
        a.xn[h] = x;
        a.woff[h] = x * a.L;
    }
}

/* kSlLanes lanes per chunk: when the feed's records (count <= cap) and output (*total <= out_cap) fit, the letters after the
 * new X become the stream's tail, and X and the position move (a final feed leaves the stream at its start) */
__global__ void acb_sl_commit_kernel(const __grid_constant__ SlArgs a, const unsigned long long *count, long long cap,
                                     const long long *total, long long out_cap) {
    if ((count && *count > (unsigned long long)cap) || (total && *total > out_cap)) return;
    const long long h = ((long long)blockIdx.x * blockDim.x + threadIdx.x) / kSlLanes;
    const int lane = threadIdx.x % kSlLanes;
    if (h >= a.n) return;
    const long long s = sl_stream(a, h);
    if (s < 0) return;
    const long long staged = (a.soff[h + 1] - a.soff[h]) / a.L, x = a.xn[h], keep = staged - x;
    const uint8_t *from = a.stage + a.soff[h] + x * a.L;
    uint8_t *to = a.tail + s * a.T * a.L;
    for (long long j = lane; j < keep * a.L; j += kSlLanes) to[j] = from[j];
    if (lane == 0) {
        const long long n = sl_chunk_bytes(a, h) / a.L;
        a.pos[s] = a.final ? 0 : a.pos[s] + n;
        a.hold[s] = a.final ? 0 : keep;
    }
}

/* Whole-word stream feeds (DESIGN section 4.15) run the pipeline above with T + 1 held letters (SlArgs::T) and these
 * kernels in place of the frontier flags (and, for find_all batches, of the selection) */
struct SwArgs {
    SlArgs a;
    uint8_t *left;                                         /* [n_streams] the letter before the held ones is a word letter */
    WordBits words;
    const int32_t *key_len;
    int leftmost;
};

/* flag[i]: record i of the staged full list lies in the feed's window and is a whole-word match.  Window: leftmost, it
 * starts before the frontier staged - (T + 1) (every record on a final feed); find_all, it ends in [hold - 1, staged - 2]
 * (staged - 1 on a final feed).  A record that starts at staged letter 0 takes its left neighbour from w.left.  A kept
 * record of a non-final feed never ends on the last staged letter, so its right neighbour is staged. */
template <int L>
__global__ void __launch_bounds__(256) acb_sw_flag_kernel(const __grid_constant__ SwArgs w, const acb_match *full,
                                                          const unsigned long long *count, long long cap, uint8_t *flag) {
    __shared__ uint32_t s_bits[8];
    const WordBits words = w.words.shared<L>(s_bits);
    const SlArgs &a = w.a;
    const long long m = min((long long)*count, cap);
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < cap; i += (long long)gridDim.x * blockDim.x) {
        bool keep = false;
        if (i < m) {
            const acb_match r = full[i];
            const long long b0 = a.soff[r.hay_id], staged = (a.soff[r.hay_id + 1] - b0) / L, s = sl_stream(a, r.hay_id);
            const long long end = r.end_index, start = end - __ldg(w.key_len + r.key_id) + 1;
            if (w.leftmost) keep = a.final || start < staged - a.T;
            else keep = end >= (s < 0 ? 0 : a.hold[s]) - 1 && end < staged - 1 + a.final;
#ifdef ACB_DEBUG
            assert(!keep || a.final || end + 1 < staged);
#endif
            if (keep) keep = !(start == 0 ? (s >= 0 && w.left[s]) : words.is_word<L>(ww_letter<L>(a.stage + b0 + (start - 1) * L)));
            if (keep && end + 1 < staged) keep = !words.is_word<L>(ww_letter<L>(a.stage + b0 + (end + 1) * L));
        }
        flag[i] = keep;
    }
}

/* out[i] = rec[i] with end_index relative to its chunk, for i < cap; *count = m */
__global__ void acb_sw_emit_kernel(const __grid_constant__ SlArgs a, const acb_match *rec, long long m, acb_match *out, long long cap,
                                   unsigned long long *count) {
    const long long first = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (first == 0) *count = (unsigned long long)m;
    for (long long i = first; i < min(m, cap); i += (long long)gridDim.x * blockDim.x) {
        acb_match r = rec[i];
        const long long s = sl_stream(a, r.hay_id);
        r.end_index = (int32_t)(r.end_index - (s < 0 ? 0 : a.hold[s]));
        out[i] = r;
    }
}

/* under the commit's condition: left[s] = staged letter X_new - 1 is a word letter (unchanged when X_new is the staged
 * start; 0 after a final feed) */
template <int L>
__global__ void acb_sw_left_kernel(const __grid_constant__ SwArgs w, const unsigned long long *count, long long cap,
                                   const long long *total, long long out_cap) {
    if ((count && *count > (unsigned long long)cap) || (total && *total > out_cap)) return;
    const SlArgs &a = w.a;
    for (long long h = (long long)blockIdx.x * blockDim.x + threadIdx.x; h < a.n; h += (long long)gridDim.x * blockDim.x) {
        const long long s = sl_stream(a, h), x = a.xn[h];
        if (s < 0) continue;
        if (a.final) w.left[s] = 0;
        else if (x > 0) w.left[s] = w.words.is_word<L>(ww_letter<L>(a.stage + a.soff[h] + (x - 1) * L));
    }
}
} // namespace

/* the feed counters d_ctr (device) and h_ctr (pinned) */
static cudaError_t streams_alloc_counters(acb_streams *ss) {
    cudaError_t e = cudaMalloc(reinterpret_cast<void **>(&ss->d_ctr), 4 * sizeof(unsigned long long));
    if (e == cudaSuccess) e = cudaMallocHost(reinterpret_cast<void **>(&ss->h_ctr), 4 * sizeof(unsigned long long));
    return e;
}

static int streams_new_leftmost(const acb_table *tb, int64_t n_streams, acb_streams **out) {
    if (!tb || !out) { acb_set_error("bad argument"); return ACB_EINVAL; }
    int rc = streams_new(tb, n_streams, 0, out);
    if (rc != ACB_OK) return rc;
    acb_streams *ss = *out;
    ss->leftmost = 1;
    const size_t n = (size_t)std::max<int64_t>(n_streams, 1);
    cudaError_t e = cudaMalloc(reinterpret_cast<void **>(&ss->d_hold), n * sizeof(long long));
    if (e == cudaSuccess) e = cudaMemset(ss->d_hold, 0, n * sizeof(long long));
    if (e == cudaSuccess) e = streams_alloc_counters(ss);
    if (e != cudaSuccess) {
        acb_set_error("allocating %lld streams: %s", (long long)n_streams, cudaGetErrorString(e));
        acb_streams_free(ss);
        *out = nullptr;
        return ACB_ECUDA;
    }
    return ACB_OK;
}

extern "C" int acb_streams_new_leftmost(const acb_table *tb, int64_t n_streams, acb_streams **out) {
    DeviceRestore keep_device;
    if (out) *out = nullptr;
    if (refuse_folded(tb, "a stream batch")) return ACB_EINVAL;
    return streams_new_leftmost(tb, n_streams, out);
}

static int streams_new_words(const acb_table *tb, int64_t n_streams, int leftmost, const uint32_t *bits, int64_t n_bits,
                             acb_streams **out) {
    if (!tb || !out) { acb_set_error("bad argument"); return ACB_EINVAL; }
    *out = nullptr;
    int rc = check_words(tb, bits, n_bits);
    if (rc != ACB_OK || (rc = streams_new_leftmost(tb, n_streams, out))) return rc;
    acb_streams *ss = *out;
    ss->leftmost = leftmost ? 1 : 0;
    ss->words = 1;
    ss->n_bits = n_bits;
    const size_t n = (size_t)std::max<int64_t>(n_streams, 1), words = ((size_t)n_bits + 31) / 32;
    cudaFree(ss->d_tail);                                  /* room for T + 1 held letters */
    ss->d_tail = nullptr;
    cudaError_t e = cudaMalloc(reinterpret_cast<void **>(&ss->d_tail), n * (ss->T + 1) * ss->L);
    if (e == cudaSuccess) e = cudaMalloc(reinterpret_cast<void **>(&ss->d_left), n);
    if (e == cudaSuccess) e = cudaMemset(ss->d_left, 0, n);
    if (e == cudaSuccess) e = cudaMalloc(reinterpret_cast<void **>(&ss->d_bits), std::max<size_t>(words, 1) * sizeof(uint32_t));
    if (e == cudaSuccess && words) e = cudaMemcpy(ss->d_bits, bits, words * sizeof(uint32_t), cudaMemcpyHostToDevice);
    if (e != cudaSuccess) {
        acb_set_error("allocating %lld streams: %s", (long long)n_streams, cudaGetErrorString(e));
        acb_streams_free(ss);
        *out = nullptr;
        return ACB_ECUDA;
    }
    return ACB_OK;
}

extern "C" int acb_streams_new_words(const acb_table *tb, int64_t n_streams, int leftmost, const uint32_t *bits, int64_t n_bits,
                                     acb_streams **out) {
    DeviceRestore keep_device;
    if (out) *out = nullptr;
    if (refuse_folded(tb, "a stream batch")) return ACB_EINVAL;
    return streams_new_words(tb, n_streams, leftmost, bits, n_bits, out);
}

/* a leftmost batch of selection `kind` (leftmost = 1) or a find_all batch (leftmost = 0), whole-word unless n_bits < 0
 * without a bitmap; of the table's kind, folded or not */
static int streams_new_kind(const acb_table *tb, int64_t n_streams, int leftmost, int kind, const uint32_t *bits, int64_t n_bits,
                            acb_streams **out) {
    if (!tb || !out) { acb_set_error("bad argument"); return ACB_EINVAL; }
    *out = nullptr;
    if (!select_kind_ok(kind)) return ACB_EINVAL;
    const bool words = n_bits >= 0 || bits;                 /* n_bits < 0 without a bitmap: no word filter */
    int rc;
    if (words) rc = streams_new_words(tb, n_streams, leftmost, bits, n_bits, out);
    else if (leftmost) rc = streams_new_leftmost(tb, n_streams, out);
    else if ((rc = streams_new(tb, n_streams, 0, out)) == ACB_OK && tb->fold) {    /* a folded find_all feed counts its full list */
        cudaError_t e = streams_alloc_counters(*out);
        if (e != cudaSuccess) {
            acb_set_error("allocating %lld streams: %s", (long long)n_streams, cudaGetErrorString(e));
            acb_streams_free(*out);
            *out = nullptr;
            return ACB_ECUDA;
        }
    }
    if (rc == ACB_OK) (*out)->kind = kind;
    return rc;
}

extern "C" int acb_streams_new_leftmost_kind(const acb_table *tb, int64_t n_streams, int kind, const uint32_t *bits, int64_t n_bits,
                                             acb_streams **out) {
    DeviceRestore keep_device;
    if (out) *out = nullptr;
    if (refuse_folded(tb, "a stream batch")) return ACB_EINVAL;
    return streams_new_kind(tb, n_streams, 1, kind, bits, n_bits, out);
}

extern "C" int acb_streams_new_folded(const acb_table *tb, int64_t n_streams, int leftmost, int kind, const uint32_t *bits, int64_t n_bits,
                                      acb_streams **out) {
    DeviceRestore keep_device;
    if (!tb || !out || (leftmost != 0 && leftmost != 1)) { acb_set_error("bad argument"); return ACB_EINVAL; }
    *out = nullptr;
    if (!tb->fold) { acb_set_error("acb_streams_new_folded takes a case-folded table (acb_table_upload_folded)"); return ACB_EINVAL; }
    return streams_new_kind(tb, n_streams, leftmost, kind, bits, n_bits, out);
}

extern "C" int acb_last_stream_leftmost_ms(float *ms, int32_t n) {
    if (!ms || n < 0 || n > 6) { acb_set_error("bad argument"); return ACB_EINVAL; }
    for (int i = 0; i < n; i++) ms[i] = g_sl_ms[i];
    return ACB_OK;
}

/* the arguments every leftmost feed (find_all_words: every find_all word feed) checks before anything runs */
static int sl_check(const acb_streams *ss, const acb_table *tb, int64_t total, const void *offsets, int64_t n, int64_t stride,
                    int *algo, bool find_all_words = false) {
    if (!ss || !tb || total < 0 || n < 0) { acb_set_error("bad argument"); return ACB_EINVAL; }
    if (find_all_words && (ss->leftmost || !ss->words)) {
        acb_set_error("not a find_all whole-word stream batch (acb_streams_new_words with leftmost = 0)");
        return ACB_EINVAL;
    }
    if (!find_all_words && !ss->leftmost) { acb_set_error("not a leftmost-longest stream batch (acb_streams_new_leftmost)"); return ACB_EINVAL; }
    int rc = streams_check_table(ss, tb);
    if (rc != ACB_OK) return rc;
    if (n > ss->n) { acb_set_error("%lld chunks for %lld streams", (long long)n, ss->n); return ACB_EINVAL; }
    if (n >= 0x7fffffffLL) { acb_set_error("2^31-1 or more chunks in one feed"); return ACB_ERANGE; }
    if (!offsets && (rc = check_stride(ss->L, total, n, stride, 0))) return rc;
    if (*algo == ACB_ALGO_AUTO) *algo = ACB_ALGO_FILTER;
    if (*algo != ACB_ALGO_FILTER && *algo != ACB_ALGO_DFA) { acb_set_error("a leftmost-longest feed takes ACB_ALGO_AUTO, _FILTER or _DFA"); return ACB_EINVAL; }
    return ACB_OK;
}

/* a replacing feed rewrites what its batch selects: the replacer's kind must be the batch's */
static int sl_kind_fits(const acb_streams *ss, const acb_replacer *r) {
    if (r->kind == ss->kind) return ACB_OK;
    acb_set_error("a replacer of selection kind %d on a stream batch of kind %d", r->kind, ss->kind);
    return ACB_EINVAL;
}

/* d_soff[0..n] <- exclusive scan of d_soff[0..n] in place; the total to the host (the one wait of the staging) */
static int sl_offsets(acb_streams *ss, long long *d, int64_t n, cudaStream_t s, long long *total) {
    size_t temp = 0;
    CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, temp, d, d, (int)(n + 1), s));
    int rc = ensure(&ss->d_tmp, &ss->tmp_cap, temp);
    if (rc) return rc;
    temp = ss->tmp_cap;
    CUDA_TRY(cub::DeviceScan::ExclusiveSum(ss->d_tmp, temp, d, d, (int)(n + 1), s));
    CUDA_TRY(cudaMemcpyAsync(ss->h_ctr + 3, d + n, sizeof(long long), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    *total = (long long)ss->h_ctr[3];
    return ACB_OK;
}

static int sl_gather(acb_streams *ss, acb_table *tb, const SlArgs &a, bool stage, const long long *doff, uint8_t *dst, long long total,
                     cudaStream_t s) {
    if (total == 0) return ACB_OK;
    const long long n_tiles = (total + kSlTile - 1) / kSlTile;
    int rc = ensure(&ss->d_ts, &ss->ts_cap, (size_t)n_tiles);
    if (rc) return rc;
    acb_sl_tiles_kernel<<<blocks(tb, n_tiles), 256, 0, s>>>(doff, a.n, total, ss->d_ts);
    if ((rc = launched("stream gather tiles"))) return rc;
    const unsigned grid = (unsigned)std::min<long long>(n_tiles, grid_sms(tb) * 8);
    if (stage) acb_sl_gather_kernel<true><<<grid, 256, 0, s>>>(a, doff, ss->d_ts, dst, total);
    else acb_sl_gather_kernel<false><<<grid, 256, 0, s>>>(a, doff, ss->d_ts, dst, total);
    return launched("stream gather");
}

static SwArgs sw_args(const acb_streams *ss, const acb_table *tb, const SlArgs &a) {
    SwArgs w;
    w.a = a; w.left = ss->d_left; w.words = {ss->d_bits, ss->n_bits}; w.key_len = tb->d_keylen; w.leftmost = ss->leftmost;
    return w;
}

/* a word feed's window and word flags over the first min(*count, fcap) records of the full list */
static int sw_flags(acb_streams *ss, acb_table *tb, const SlArgs &a, long long fcap, cudaStream_t s) {
    const SwArgs w = sw_args(ss, tb, a);
    with_width(ss->L, [&](auto l) {
        acb_sw_flag_kernel<decltype(l)::value><<<blocks(tb, fcap), 256, 0, s>>>(w, ss->d_full, ss->d_ctr, fcap, ss->d_flag);
    });
    return launched("stream word flags");
}

/* A folded word feed's m kept records (ss->d_settled) with every alias of their key added, into ss->d_full, grown until
 * they fit (one wait for their number, counted in d_ctr[2]); *m becomes that number */
static int sw_expand(acb_streams *ss, acb_table *tb, unsigned long long *m, cudaStream_t s) {
    int rc = ensure(&ss->d_full, &ss->full_cap, (size_t)*m);
    for (; rc == ACB_OK;) {
        const int64_t cap = (int64_t)std::min<size_t>(ss->full_cap, 0x7fffffffULL);
        if ((rc = acb_expand_aliases_device(tb, ss->d_settled, (int64_t)*m, ss->d_full, cap, reinterpret_cast<int64_t *>(ss->d_ctr + 2), s)))
            return rc;
        CUDA_TRY(cudaMemcpyAsync(ss->h_ctr + 2, ss->d_ctr + 2, sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
        CUDA_TRY(cudaStreamSynchronize(s));
        if (ss->h_ctr[2] <= (unsigned long long)cap) break;
        if (ss->h_ctr[2] > 0x7fffffffULL) { acb_set_error("more than 2^31-1 matches in one feed"); return ACB_ERANGE; }
        rc = ensure(&ss->d_full, &ss->full_cap, (size_t)ss->h_ctr[2]);
    }
    if (rc != ACB_OK) return rc;
    *m = ss->h_ctr[2];
    return ensure(&ss->d_settled, &ss->settled_cap, (size_t)*m);        /* the sort's second buffer */
}

/* a find_all word feed's m kept records (ss->d_settled, staged coordinates; on a folded table with aliases, expanded
 * first) in the reference order -- chunk, end, longest key first, a group of case variants in ascending id (the sort is
 * stable) -- and rebased to their chunks into d_out (the first cap of them); *d_count = their number */
static int sw_order(acb_streams *ss, acb_table *tb, const SlArgs &a, unsigned long long m, long long staged, acb_match *d_out,
                    int64_t cap, unsigned long long *d_count, cudaStream_t s) {
    if (m == 0) return ACB_OK;                             /* *d_count is 0 already */
    acb_match *in = ss->d_settled, *mid = ss->d_full;
    int rc;
    if (tb->n_alias) {
        if ((rc = sw_expand(ss, tb, &m, s))) return rc;
        in = ss->d_full;
        mid = ss->d_settled;
    }
    const SortKey k = sort_key(tb, a.n, staged / a.L);
    if ((rc = ensure(&ss->d_keys, &ss->keys_cap, 2 * (size_t)m))) return rc;
    unsigned long long *k0 = ss->d_keys, *k1 = ss->d_keys + m;
    size_t temp = 0;
    CUDA_TRY(cub::DeviceRadixSort::SortPairs(nullptr, temp, k0, k1, in, mid, (int)m, 0, 64, s));
    if ((rc = ensure(&ss->d_tmp, &ss->tmp_cap, temp))) return rc;
    acb_match *sorted = k.bits() <= 64 ? mid : in;          /* two passes go through mid */
    if ((rc = sort_records<kKeyEnd, kKeyEndLow>(tb, k, in, mid, sorted, (long long)m, k0, k1, ss->d_tmp, ss->tmp_cap, s,
                                  "stream word sort key")))
        return rc;
    acb_sw_emit_kernel<<<blocks(tb, m), 256, 0, s>>>(a, sorted, (long long)m, d_out, cap, d_count);
    return launched("stream word emit");
}

/* the left-neighbour flags of the fed streams, under the commit's condition */
static int sw_left(acb_streams *ss, acb_table *tb, const SlArgs &a, const unsigned long long *count, long long cap,
                   const long long *total, long long out_cap, cudaStream_t s) {
    const SwArgs w = sw_args(ss, tb, a);
    with_width(ss->L, [&](auto l) { acb_sw_left_kernel<decltype(l)::value><<<blocks(tb, a.n), 256, 0, s>>>(w, count, cap, total, out_cap); });
    return launched("stream word edge");
}

/* The leftmost feed on DEVICE buffers, both forms.  r == nullptr: the chosen records go to d_out (cap, *d_count,
 * end_index relative to the chunk); else the decided windows are rewritten into d_rout (d_rout_off, *d_rtotal,
 * out_cap).  Waits for the staged size, for the full list's size, and (replacing) for the windows' size. */
static int sl_feed(acb_streams *ss, acb_table *tb, acb_replacer *r, const uint8_t *d_chunks, int64_t total, const int64_t *d_off,
                   int64_t n, int64_t stride, const int32_t *d_ids, int final, acb_match *d_out, int64_t cap, int64_t *d_count,
                   int64_t *d_rout_off, uint8_t *d_rout, int64_t out_cap, int64_t *d_rtotal, cudaStream_t s, int algo) {
    int rc;
    for (float &v : g_sl_ms) v = 0.f;
    if (ss->fold) g_fold_ms[0] = g_fold_ms[1] = 0.f;
    CUDA_TRY(cudaSetDevice(ss->device));
    if (!r) CUDA_TRY(cudaMemsetAsync(d_count, 0, sizeof(int64_t), s));
    if (n == 0) {
        if (r) CUDA_TRY(cudaMemsetAsync(d_rout_off, 0, sizeof(int64_t), s));
        if (r) CUDA_TRY(cudaMemsetAsync(d_rtotal, 0, sizeof(int64_t), s));
        return ACB_OK;
    }
    if (total && (reinterpret_cast<uintptr_t>(d_chunks) & 15)) { acb_set_error("d_chunks must be 16-byte aligned"); return ACB_EINVAL; }
    const size_t N = (size_t)n;
    if ((rc = ensure(&ss->d_soff, &ss->soff_cap, N + 1)) || (rc = ensure(&ss->d_aux, &ss->aux_cap, 3 * N + 1))) return rc;
    SlArgs a;
    memset(&a, 0, sizeof(a));
    a.ids = d_ids; a.n_streams = ss->n; a.pos = ss->d_pos; a.hold = ss->d_hold; a.tail = ss->d_tail; a.T = ss->T + ss->words; a.L = ss->L;
    a.chunks = d_chunks; a.off = reinterpret_cast<const long long *>(d_off); a.stride = stride; a.n = n;
    a.soff = ss->d_soff; a.last = ss->d_aux; a.xn = ss->d_aux + N; a.woff = ss->d_aux + 2 * N; a.final = final ? 1 : 0;
    const unsigned g_chunks = blocks(tb, n + 1);
    /* 1. stage */
    acb_sl_len_kernel<<<g_chunks, 256, 0, s>>>(a);
    if ((rc = launched("stream staged lengths"))) return rc;
    long long staged = 0;
    if ((rc = sl_offsets(ss, ss->d_soff, n, s, &staged))) return rc;
    if ((rc = ensure(&ss->d_stage, &ss->stage_cap, (size_t)staged + 64))) return rc;
    a.stage = ss->d_stage;
    if ((rc = timing_mark(&ss->ev[0], s)) || (rc = sl_gather(ss, tb, a, true, ss->d_soff, ss->d_stage, staged, s)) || (rc = timing_mark(&ss->ev[1], s))) return rc;
    /* 2. scan and 3. the frontier filter; the full list grows until it fits */
    const int64_t *soff = reinterpret_cast<const int64_t *>(ss->d_soff);
    unsigned long long m = 0;
    for (;;) {
        size_t fcap = std::max<size_t>(ss->full_cap, 4096);
        if (fcap > 0x7fffffffULL) fcap = 0x7fffffffULL;
        if ((rc = ensure(&ss->d_full, &ss->full_cap, fcap)) || (rc = ensure(&ss->d_settled, &ss->settled_cap, fcap)) ||
            (rc = ensure(&ss->d_flag, &ss->flag_cap, fcap)))
            return rc;
        fcap = std::min<size_t>(ss->full_cap, 0x7fffffffULL);
        CUDA_TRY(cudaMemsetAsync(ss->d_ctr, 0, 4 * sizeof(unsigned long long), s));
        if ((rc = timing_mark(&ss->ev[2], s))) return rc;
        if (staged && (rc = acb_scan_device(tb, ss->d_stage, staged, soff, n, 0, ss->d_full, (int64_t)fcap,
                                            reinterpret_cast<int64_t *>(ss->d_ctr), s, algo)))
            return rc;
        if ((rc = timing_mark(&ss->ev[3], s)) || (rc = timing_mark(&ss->ev[4], s))) return rc;
        if (ss->words) {
            if ((rc = sw_flags(ss, tb, a, (long long)fcap, s))) return rc;
        } else {
            acb_sl_flag_kernel<<<blocks(tb, (long long)fcap), 256, 0, s>>>(a, ss->d_full, ss->d_ctr, (long long)fcap, tb->d_keylen, ss->d_flag);
            if ((rc = launched("stream frontier flags"))) return rc;
        }
        size_t temp = 0;
        CUDA_TRY(cub::DeviceSelect::Flagged(nullptr, temp, ss->d_full, ss->d_flag, ss->d_settled, ss->d_ctr + 1, (int)fcap, s));
        if ((rc = ensure(&ss->d_tmp, &ss->tmp_cap, temp))) return rc;
        temp = ss->tmp_cap;
        CUDA_TRY(cub::DeviceSelect::Flagged(ss->d_tmp, temp, ss->d_full, ss->d_flag, ss->d_settled, ss->d_ctr + 1, (int)fcap, s));
        if ((rc = timing_mark(&ss->ev[5], s))) return rc;
        CUDA_TRY(cudaMemcpyAsync(ss->h_ctr, ss->d_ctr, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
        CUDA_TRY(cudaStreamSynchronize(s));
        if (ss->h_ctr[0] <= fcap) { m = ss->h_ctr[1]; break; }
        if (ss->h_ctr[0] > 0x7fffffffULL) { acb_set_error("more than 2^31-1 matches in one feed"); return ACB_ERANGE; }
        if ((rc = ensure(&ss->d_full, &ss->full_cap, (size_t)ss->h_ctr[0]))) return rc;
    }
    if ((rc = timing_ms(ss->ev[0], ss->ev[1], &g_sl_ms[0])) || (rc = timing_ms(ss->ev[2], ss->ev[3], &g_sl_ms[1])) ||
        (rc = timing_ms(ss->ev[4], ss->ev[5], &g_sl_ms[2])))
        return rc;
    /* 4. select */
    acb_match *chosen = d_out;
    int64_t ccap = cap;
    unsigned long long *ccount = reinterpret_cast<unsigned long long *>(d_count);
    if (r) {
        if ((rc = ensure(&ss->d_chosen, &ss->chosen_cap, (size_t)std::max<unsigned long long>(m, 1)))) return rc;
        chosen = ss->d_chosen; ccap = (int64_t)m; ccount = ss->d_ctr + 2;
    }
    const int64_t max_letters = std::max<int64_t>(staged / ss->L, 1);
    if ((rc = timing_mark(&ss->ev[6], s))) return rc;
    if (!ss->leftmost) {                                   /* a find_all word feed returns every kept record, ordered */
        if ((rc = sw_order(ss, tb, a, m, staged, d_out, cap, ccount, s))) return rc;
    } else if (m && (rc = leftmost_select(tb, ss->kind, ss->d_settled, (int64_t)m, n, max_letters, chosen, ccap,
                                          reinterpret_cast<int64_t *>(ccount), s))) {
        return rc;
    }
    if ((rc = timing_mark(&ss->ev[7], s))) return rc;
    /* 5. the new X per chunk, and the windows of a replacing feed */
    CUDA_TRY(cudaMemsetAsync(a.last, 0xff, N * sizeof(long long), s));
    if (m && ss->leftmost) {
        acb_sl_last_kernel<<<blocks(tb, (long long)m), 256, 0, s>>>(a, chosen, ccount, ccap, r ? 0 : 1);
        if ((rc = launched("stream last chosen"))) return rc;
    }
    acb_sl_frontier_kernel<<<g_chunks, 256, 0, s>>>(a);
    if ((rc = launched("stream frontier"))) return rc;
    if (r) {
        long long wtotal = 0;
        if ((rc = sl_offsets(ss, a.woff, n, s, &wtotal))) return rc;
        if ((rc = ensure(&ss->d_win, &ss->win_cap, (size_t)wtotal + 64))) return rc;
        if ((rc = timing_mark(&ss->ev[8], s)) || (rc = sl_gather(ss, tb, a, false, a.woff, ss->d_win, wtotal, s)) || (rc = timing_mark(&ss->ev[9], s))) return rc;
        if ((rc = acb_replace_device(r, tb, ss->d_win, wtotal, reinterpret_cast<const int64_t *>(a.woff), n, 0, chosen, ccap,
                                     reinterpret_cast<const int64_t *>(ccount), d_rout_off, d_rout, out_cap, d_rtotal, s)))
            return rc;
    }
    /* 6. commit */
    if ((rc = timing_mark(&ss->ev[10], s))) return rc;
    if (ss->words && (rc = sw_left(ss, tb, a, r ? nullptr : ccount, ccap, r ? reinterpret_cast<const long long *>(d_rtotal) : nullptr,
                                   out_cap, s)))
        return rc;
    acb_sl_commit_kernel<<<(unsigned)((n * kSlLanes + 255) / 256), 256, 0, s>>>(a, r ? nullptr : ccount, ccap,
                                                                          r ? reinterpret_cast<const long long *>(d_rtotal) : nullptr, out_cap);
    if ((rc = launched("stream commit")) || (rc = timing_mark(&ss->ev[11], s)) || (rc = timing_ms(ss->ev[6], ss->ev[7], &g_sl_ms[3])) ||
        (r && (rc = timing_ms(ss->ev[8], ss->ev[9], &g_sl_ms[4]))))
        return rc;
    return timing_ms(ss->ev[10], ss->ev[11], &g_sl_ms[5]);
}

static int sl_feed_device(acb_streams *ss, acb_table *tb, const uint8_t *d_chunks, int64_t total_bytes, const int64_t *d_offsets,
                          int64_t n_chunks, int64_t stride_bytes, const int32_t *d_ids, int final, acb_match *d_out, int64_t cap,
                          int64_t *d_count, void *stream, int algo, bool find_all_words) {
    int rc = sl_check(ss, tb, total_bytes, d_offsets, n_chunks, stride_bytes, &algo, find_all_words);
    if (rc) return rc;
    if (!d_count || cap < 0 || (cap > 0 && !d_out) || (total_bytes && !d_chunks)) { acb_set_error("bad argument"); return ACB_EINVAL; }
    return sl_feed(ss, tb, nullptr, d_chunks, total_bytes, d_offsets, n_chunks, stride_bytes, d_ids, final, d_out, cap, d_count,
                   nullptr, nullptr, 0, nullptr, reinterpret_cast<cudaStream_t>(stream), algo);
}

extern "C" int acb_streams_feed_leftmost_device(acb_streams *ss, acb_table *tb, const uint8_t *d_chunks, int64_t total_bytes,
                                                const int64_t *d_offsets, int64_t n_chunks, int64_t stride_bytes, const int32_t *d_ids,
                                                int final, acb_match *d_out, int64_t cap, int64_t *d_count, void *stream, int algo) {
    DeviceRestore keep_device;
    return sl_feed_device(ss, tb, d_chunks, total_bytes, d_offsets, n_chunks, stride_bytes, d_ids, final, d_out, cap, d_count, stream,
                          algo, false);
}

extern "C" int acb_streams_feed_words_device(acb_streams *ss, acb_table *tb, const uint8_t *d_chunks, int64_t total_bytes,
                                             const int64_t *d_offsets, int64_t n_chunks, int64_t stride_bytes, const int32_t *d_ids,
                                             int final, acb_match *d_out, int64_t cap, int64_t *d_count, void *stream, int algo) {
    DeviceRestore keep_device;
    return sl_feed_device(ss, tb, d_chunks, total_bytes, d_offsets, n_chunks, stride_bytes, d_ids, final, d_out, cap, d_count, stream,
                          algo, true);
}

extern "C" int acb_streams_replace_device(acb_streams *ss, acb_replacer *r, acb_table *tb, const uint8_t *d_chunks, int64_t total_bytes,
                                          const int64_t *d_offsets, int64_t n_chunks, int64_t stride_bytes, const int32_t *d_ids, int final,
                                          int64_t *d_out_offsets, uint8_t *d_out, int64_t out_cap, int64_t *d_total, void *stream, int algo) {
    DeviceRestore keep_device;
    int rc = sl_check(ss, tb, total_bytes, d_offsets, n_chunks, stride_bytes, &algo);
    if (rc) return rc;
    if (!r || !d_out_offsets || !d_total || out_cap < 0 || (out_cap && !d_out) || (total_bytes && !d_chunks)) { acb_set_error("bad argument"); return ACB_EINVAL; }
    if ((rc = rp_fits(r, tb)) || (rc = sl_kind_fits(ss, r))) return rc;
    if (reinterpret_cast<uintptr_t>(d_out) & 15) { acb_set_error("d_out must be 16-byte aligned"); return ACB_EINVAL; }
    return sl_feed(ss, tb, r, d_chunks, total_bytes, d_offsets, n_chunks, stride_bytes, d_ids, final, nullptr, 0, nullptr,
                   d_out_offsets, d_out, out_cap, d_total, reinterpret_cast<cudaStream_t>(stream), algo);
}

/* a host feed's first step: ids and offsets checked, chunks (+ offsets, ids) uploaded to the table's workspace */
static int sl_upload(acb_streams *ss, acb_table *tb, const uint8_t *chunks, int64_t total, const int64_t *offsets, int64_t n,
                     const int32_t *ids, const int64_t **d_off) {
    int rc;
    if (ids && (rc = check_ids(ss, ids, n))) return rc;
    if (offsets && (rc = check_offsets(ss->L, offsets, n, total))) return rc;
    if ((rc = upload_batch(tb, chunks, total, offsets, n, d_off))) return rc;
    return upload_ids(ss, ids, n, tb->stream);
}

static int sl_feed_host(acb_streams *ss, acb_table *tb, const uint8_t *chunks, int64_t total_bytes, const int64_t *offsets,
                        int64_t n_chunks, int64_t stride_bytes, const int32_t *ids, int final, acb_match *out, int64_t cap, int64_t *n_found,
                        int algo, bool find_all_words) {
    int rc = sl_check(ss, tb, total_bytes, offsets, n_chunks, stride_bytes, &algo, find_all_words);
    if (rc) return rc;
    if (!n_found || cap < 0 || (total_bytes && !chunks)) { acb_set_error("bad argument"); return ACB_EINVAL; }
    *n_found = 0;
    tb->h_out_n = 0;
    const int64_t *d_off = nullptr;
    if ((rc = sl_upload(ss, tb, chunks, total_bytes, offsets, n_chunks, ids, &d_off)) ||
        (rc = ensure(&tb->w_out, &tb->w_out_cap, (size_t)std::max<int64_t>(cap, 1))))
        return rc;
    cudaStream_t s = tb->stream;
    if ((rc = sl_feed(ss, tb, nullptr, tb->w_hay, total_bytes, d_off, n_chunks, stride_bytes, ids ? ss->d_ids : nullptr, final, tb->w_out, cap,
                      reinterpret_cast<int64_t *>(tb->w_count), nullptr, nullptr, 0, nullptr, s, algo)))
        return rc;
    return read_back(tb, tb->w_count, tb->w_out, cap, 0, n_chunks, 0, out, n_found, s);
}

extern "C" int acb_streams_feed_leftmost_host(acb_streams *ss, acb_table *tb, const uint8_t *chunks, int64_t total_bytes,
                                              const int64_t *offsets, int64_t n_chunks, int64_t stride_bytes, const int32_t *ids, int final,
                                              acb_match *out, int64_t cap, int64_t *n_found, int algo) {
    DeviceRestore keep_device;
    return sl_feed_host(ss, tb, chunks, total_bytes, offsets, n_chunks, stride_bytes, ids, final, out, cap, n_found, algo, false);
}

extern "C" int acb_streams_feed_words_host(acb_streams *ss, acb_table *tb, const uint8_t *chunks, int64_t total_bytes,
                                           const int64_t *offsets, int64_t n_chunks, int64_t stride_bytes, const int32_t *ids, int final,
                                           acb_match *out, int64_t cap, int64_t *n_found, int algo) {
    DeviceRestore keep_device;
    return sl_feed_host(ss, tb, chunks, total_bytes, offsets, n_chunks, stride_bytes, ids, final, out, cap, n_found, algo, true);
}

extern "C" int acb_streams_replace_host(acb_streams *ss, acb_replacer *r, acb_table *tb, const uint8_t *chunks, int64_t total_bytes,
                                        const int64_t *offsets, int64_t n_chunks, int64_t stride_bytes, const int32_t *ids, int final,
                                        int algo, int64_t *out_offsets, uint8_t *out, int64_t out_cap, int64_t *total) {
    DeviceRestore keep_device;
    int rc = sl_check(ss, tb, total_bytes, offsets, n_chunks, stride_bytes, &algo);
    if (rc) return rc;
    if (!r || !out_offsets || !total || out_cap < 0 || (out_cap && !out) || (total_bytes && !chunks)) { acb_set_error("bad argument"); return ACB_EINVAL; }
    if ((rc = rp_fits(r, tb)) || (rc = sl_kind_fits(ss, r))) return rc;
    *total = 0;
    const int64_t *d_off = nullptr;
    if ((rc = sl_upload(ss, tb, chunks, total_bytes, offsets, n_chunks, ids, &d_off))) return rc;
    cudaStream_t s = tb->stream;
    if ((rc = ensure(&tb->r_off, &tb->r_off_cap, (size_t)n_chunks + 2))) return rc;
    const int64_t guess = total_bytes + total_bytes / 4 + n_chunks * (int64_t)(ss->T + ss->words) * ss->L + 4096;
    if ((rc = ensure(&tb->r_out, &tb->r_out_cap, (size_t)std::max<int64_t>(std::min(out_cap, guess), 16)))) return rc;
    for (;;) {                                             /* an output that fits out_cap but not the device buffer: grow, repeat */
        const int64_t dev_cap = std::min<int64_t>(out_cap, (int64_t)tb->r_out_cap);
        if ((rc = sl_feed(ss, tb, r, tb->w_hay, total_bytes, d_off, n_chunks, stride_bytes, ids ? ss->d_ids : nullptr, final, nullptr, 0,
                          nullptr, reinterpret_cast<int64_t *>(tb->r_off), tb->r_out, dev_cap, reinterpret_cast<int64_t *>(tb->r_off + n_chunks + 1),
                          s, algo)))
            return rc;
        CUDA_TRY(cudaMemcpyAsync(out_offsets, tb->r_off, (size_t)(n_chunks + 1) * sizeof(int64_t), cudaMemcpyDeviceToHost, s));
        CUDA_TRY(cudaMemcpyAsync(total, tb->r_off + n_chunks + 1, sizeof(int64_t), cudaMemcpyDeviceToHost, s));
        CUDA_TRY(cudaStreamSynchronize(s));
        if (*total > out_cap) {
            acb_set_error("replacement: room for %lld bytes, output %lld", (long long)out_cap, (long long)*total);
            return ACB_EOVERFLOW;
        }
        if (*total <= dev_cap) break;
        if ((rc = ensure(&tb->r_out, &tb->r_out_cap, (size_t)*total))) return rc;
    }
    if (*total) CUDA_TRY(cudaMemcpyAsync(out, tb->r_out, (size_t)*total, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    return ACB_OK;
}

/* ------------------------------------------------------------ UTF-8 batches (DESIGN section 4.20) */
/* A batch of UTF-8 haystacks decoded to letters of 1 or 4 bytes, byte by byte and in parallel: a byte starts a letter
 * unless it is a continuation byte (0x80-0xBF) that the nearest non-continuation byte at most 3 bytes before it, in its
 * haystack, covers with its maximal valid prefix (Unicode Table 3-7, never past the haystack's end).  A letter whose
 * maximal prefix is not a whole sequence is invalid and decodes to U+FFFD.  Haystack by haystack this is CPython's
 * bytes.decode("utf-8", "replace"), and the first invalid letter is its strict error: start at the letter, end after
 * its prefix.
 * Pass 1 (acb_utf8_decode_kernel) keeps the white-space compaction's metadata -- a start mask per 32-byte group, uint16
 * group prefixes within a tile, int64 tile prefixes from a decoupled look-back (CompactMeta, kept_before) -- and
 * reduces the largest letter and the first error; acb_utf8_offsets_kernel gives each haystack's first letter, the
 * longest haystack and the letter total.  Pass 2 (acb_utf8_write_kernel) classifies the bytes again, decodes every
 * start and stores it at its rank, staged per tile in shared memory so the stores are coalesced. */
namespace {
constexpr int kU8Stage = 1024;                            /* haystack offsets around a tile staged in shared memory */
constexpr int kU8Look = 36;                               /* bytes past a group whose haystack starts a group needs */

struct U8Args {
    const uint8_t *in;            /* 16-byte aligned */
    long long total;
    const long long *off;         /* n_hay + 1 byte offsets, or nullptr: rows of `stride` bytes */
    long long stride, n_hay;
    uint32_t *mask;
    uint16_t *gpre;
    long long *tile_pre;          /* [n_tiles + 1] */
    unsigned long long *status;   /* [n_tiles], zeroed */
    unsigned int *ctr;            /* zeroed */
    unsigned long long *err;      /* first invalid letter: start << 2 | (prefix length - 1); all ones for none */
    long long *loff;              /* [n_hay + 1]: first letter of each haystack */
    long long *info;              /* [5]: letters, largest letter, longest haystack in letters, error start, error end */
    long long n_tiles;
    int strict;
};

/* byte i (-4 <= i < 36) of a group's window: w[0] holds the 4 bytes before the group, w[1..8] its 32, w[9] the 4 after */
__device__ __forceinline__ uint32_t u8_at(const uint32_t (&w)[10], int i) { return (w[(i + 4) >> 2] >> (8 * ((i + 4) & 3))) & 255u; }

/* the window of the group at p0 (a multiple of 32), zero outside the batch */
__device__ __forceinline__ void u8_load(const uint8_t *in, long long total, long long p0, uint32_t (&w)[10]) {
    if (p0 >= 4 && p0 + 36 <= total) {
        const uint4 *src = reinterpret_cast<const uint4 *>(in + p0);
        const uint4 v0 = src[0], v1 = src[1];
        w[0] = __ldg(reinterpret_cast<const uint32_t *>(in + p0) - 1);
        w[1] = v0.x; w[2] = v0.y; w[3] = v0.z; w[4] = v0.w; w[5] = v1.x; w[6] = v1.y; w[7] = v1.z; w[8] = v1.w;
        w[9] = __ldg(reinterpret_cast<const uint32_t *>(in + p0 + 32));
        return;
    }
#pragma unroll
    for (int k = 0; k < 10; k++) w[k] = 0;
#pragma unroll
    for (int i = -4; i < 36; i++)                          /* unrolled: w stays in registers */
        if (p0 + i >= 0 && p0 + i < total) w[(i + 4) >> 2] |= (uint32_t)in[p0 + i] << (8 * ((i + 4) & 3));
}

/* haystack offsets read from the tile's staged copy when it fits, else from global memory */
struct U8Offs {
    const long long *s, *g;
    long long base;
    bool staged;
    __device__ __forceinline__ long long at(long long h) const { return staged ? s[h - base] : __ldg(g + h); }
    /* the first h in [lo, hi) with at(h) > x (upper) or >= x (lower), else hi */
    __device__ __forceinline__ long long first(long long lo, long long hi, long long x, bool upper) const {
        while (lo < hi) {
            const long long mid = (lo + hi) >> 1, v = at(mid);
            if (v < x || (upper && v == x)) lo = mid + 1; else hi = mid;
        }
        return lo;
    }
};

/* The haystack starts among bytes p0 - 3 .. p0 + 36 as bits 1 .. 40 (bit 4 + i: a haystack starts at byte p0 + i); the
 * batch's end counts as one.  o: the tile's offsets, holding every offset in [t0 - 3, t0 + kCmpTile + kU8Look] in
 * [lo, hi) */
__device__ __forceinline__ unsigned long long u8_bounds(const U8Args &a, const U8Offs &o, long long lo, long long hi, long long p0) {
    unsigned long long b = 0;
    if (!a.off) {
        for (long long x = (max(p0 - 3, 0LL) + a.stride - 1) / a.stride * a.stride; x <= p0 + kU8Look && x <= a.total; x += a.stride)
            b |= 1ULL << (x - p0 + 4);
        return b;
    }
    for (long long h = o.first(lo, hi, p0 - 3, false); h < hi;) {
        const long long x = o.at(h);
        if (x > p0 + kU8Look) break;
        b |= 1ULL << (x - p0 + 4);
        h = o.first(h + 1, hi, x, true);                   /* past the empty haystacks that start there too */
    }
    return b;
}

/* The tile's haystack offsets, staged in shared memory when they fit (ragged batches; block-wide, every thread calls) */
__device__ __forceinline__ U8Offs u8_stage(const U8Args &a, long long t0, long long *s_off, long long *s_range, long long *lo, long long *hi) {
    U8Offs o{s_off, a.off, 0, false};
    if (!a.off) return o;
    if (threadIdx.x == 0) {
        U8Offs g{nullptr, a.off, 0, false};
        s_range[0] = g.first(0, a.n_hay + 1, max(t0 - 3, 0LL), false);
        s_range[1] = g.first(s_range[0], a.n_hay + 1, min(t0 + kCmpTile + kU8Look, a.total), true);
    }
    __syncthreads();
    *lo = s_range[0];
    *hi = s_range[1];
    if (*hi - *lo <= kU8Stage) {
        for (long long i = threadIdx.x; i < *hi - *lo; i += blockDim.x) s_off[i] = __ldg(a.off + *lo + i);
        o.base = *lo;
        o.staged = true;
    }
    __syncthreads();
    return o;
}

/* The maximal valid prefix of the sequence that byte i of the window leads (bnd: u8_bounds): its length when it is a
 * whole sequence, with *cp its code point; minus its length when it is not, with *cp U+FFFD */
__device__ __forceinline__ int u8_prefix(const uint32_t (&w)[10], int i, unsigned long long bnd, uint32_t *cp) {
    const uint32_t b0 = u8_at(w, i);
    if (b0 < 0x80u) { *cp = b0; return 1; }
    const int need = b0 < 0xC2u ? 0 : b0 < 0xE0u ? 2 : b0 < 0xF0u ? 3 : b0 < 0xF5u ? 4 : 0;
    *cp = 0xFFFDu;
    if (!need) return -1;
    const unsigned long long after = bnd >> (i + 5);       /* haystack starts after byte i */
    const int avail = after ? __ffsll((long long)after) : 64;
    const uint32_t b1 = u8_at(w, i + 1), b2 = u8_at(w, i + 2), b3 = u8_at(w, i + 3);
    const uint32_t lo = b0 == 0xE0u ? 0xA0u : b0 == 0xF0u ? 0x90u : 0x80u, hi = b0 == 0xEDu ? 0x9Fu : b0 == 0xF4u ? 0x8Fu : 0xBFu;
    int k = 1;
    if (avail > 1 && b1 >= lo && b1 <= hi) {
        k = 2;
        if (need > 2 && avail > 2 && (b2 & 0xC0u) == 0x80u) {
            k = 3;
            if (need > 3 && avail > 3 && (b3 & 0xC0u) == 0x80u) k = 4;
        }
    }
    if (k < need) return -k;
    *cp = need == 2 ? (b0 & 0x1Fu) << 6 | (b1 & 0x3Fu)
        : need == 3 ? (b0 & 0x0Fu) << 12 | (b1 & 0x3Fu) << 6 | (b2 & 0x3Fu)
                    : (b0 & 0x07u) << 18 | (b1 & 0x3Fu) << 12 | (b2 & 0x3Fu) << 6 | (b3 & 0x3Fu);
    return k;
}

/* bit j: byte j of the group starts a letter; bytes from `valid` on (past the batch) never do */
__device__ __forceinline__ uint32_t u8_starts(const uint32_t (&w)[10], unsigned long long bnd, int valid) {
    uint32_t keep = 0;
#pragma unroll
    for (int j = 0; j < 32; j++) {
        bool start = true;
        if ((u8_at(w, j) & 0xC0u) == 0x80u) {
#pragma unroll
            for (int d = 1; d <= 3; d++) {
                const int q = j - d;
                if ((bnd >> (q + 5)) & ((1ULL << d) - 1)) break;      /* a haystack starts between the lead and byte j */
                if ((u8_at(w, q) & 0xC0u) == 0x80u) continue;
                uint32_t cp;
                start = abs(u8_prefix(w, q, bnd, &cp)) <= d;
                break;
            }
        }
        if (start && j < valid) keep |= 1u << j;
    }
    return keep;
}

__device__ __forceinline__ bool u8_ascii(const uint32_t (&w)[10]) {
    return ((w[1] | w[2] | w[3] | w[4] | w[5] | w[6] | w[7] | w[8]) & 0x80808080u) == 0;
}

__global__ void __launch_bounds__(kCmpThreads) acb_utf8_decode_kernel(const __grid_constant__ U8Args a) {
    using Scan = cub::BlockScan<int, kCmpThreads>;
    __shared__ typename Scan::TempStorage scan_tmp;
    __shared__ long long s_off[kU8Stage];
    __shared__ long long s_tile, s_range[2];
    __shared__ unsigned int s_max;
    if (threadIdx.x == 0) { s_tile = atomicAdd(a.ctr, 1u); s_max = 0; }   /* in claim order: every earlier tile is running or done */
    __syncthreads();
    const long long tile = s_tile, t0 = tile * kCmpTile, p0 = t0 + (long long)threadIdx.x * 32;
    long long lo = 0, hi = 0;
    const U8Offs o = u8_stage(a, t0, s_off, s_range, &lo, &hi);
    uint32_t w[10];
    u8_load(a.in, a.total, p0, w);
    const int valid = (int)max(min(32LL, a.total - p0), 0LL);
    uint32_t keep, mx = 0;
    unsigned long long err = ~0ULL;
    if (u8_ascii(w)) {
        keep = valid == 32 ? ~0u : (1u << valid) - 1u;
        uint32_t m = __vmaxu4(__vmaxu4(__vmaxu4(w[1], w[2]), __vmaxu4(w[3], w[4])), __vmaxu4(__vmaxu4(w[5], w[6]), __vmaxu4(w[7], w[8])));
        m = __vmaxu4(m, m >> 16);
        mx = __vmaxu4(m, m >> 8) & 255u;                   /* bytes past the batch are zero */
    } else {
        const unsigned long long bnd = u8_bounds(a, o, lo, hi, p0);
        keep = u8_starts(w, bnd, valid);
#pragma unroll
        for (int j = 0; j < 32; j++) {
            if (!((keep >> j) & 1)) continue;
            uint32_t cp;
            const int k = u8_prefix(w, j, bnd, &cp);
            mx = max(mx, cp);
            if (k < 0 && err == ~0ULL) err = (unsigned long long)(p0 + j) << 2 | (unsigned long long)(-k - 1);
        }
    }
    int pre, agg;
    Scan(scan_tmp).ExclusiveSum(__popc(keep), pre, agg);
    const long long g = tile * kCmpThreads + threadIdx.x;
    a.mask[g] = keep;
    a.gpre[g] = (uint16_t)pre;
    mx = __reduce_max_sync(kFull, mx);
    if ((threadIdx.x & 31) == 0 && mx) atomicMax(&s_max, mx);
    if (a.strict && err != ~0ULL) atomicMin(a.err, err);
    if (threadIdx.x == 0) {                                /* decoupled look-back over the tiles before this one */
        long long base = 0;
        if (tile == 0) {
            atomicExch(a.status, kLbPre | (unsigned long long)agg);
        } else {
            atomicExch(a.status + tile, kLbAgg | (unsigned long long)agg);
            for (long long i = tile - 1;; --i) {
                unsigned long long st;
                while ((st = *reinterpret_cast<volatile unsigned long long *>(a.status + i)) == 0) {}
                base += (long long)(st & kLbVal);
                if (st & kLbPre) break;
            }
            atomicExch(a.status + tile, kLbPre | (unsigned long long)(base + agg));
        }
        a.tile_pre[tile] = base;
        if (tile == a.n_tiles - 1) a.tile_pre[a.n_tiles] = base + agg;
    }
    __syncthreads();
    if (threadIdx.x == 0 && s_max) atomicMax(a.info + 1, (long long)s_max);
}
} // namespace

namespace {
/* a.loff[h] = first letter of haystack h (h = 0 .. n_hay); the longest haystack, the letter total and the error into
 * a.info */
__global__ void acb_utf8_offsets_kernel(const CompactMeta m, const __grid_constant__ U8Args a) {
    const long long h = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (h > a.n_hay) return;
    const long long s = kept_before(m, hay_start(a.off, a.stride, h));
    a.loff[h] = s;
    if (h < a.n_hay) {
        const long long len = kept_before(m, hay_start(a.off, a.stride, h + 1)) - s;
        if (len) atomicMax(a.info + 2, len);
        return;
    }
    a.info[0] = s;
    const unsigned long long e = *a.err;
    a.info[3] = e == ~0ULL ? -1 : (long long)(e >> 2);
    a.info[4] = e == ~0ULL ? -1 : (long long)(e >> 2) + (long long)(e & 3) + 1;
}

/* Pass 2: the letters of tile blockIdx.x at W bytes each into out (from letter tile_pre[tile] on), and out_off[h] =
 * W * loff[h] over a grid-stride loop.  Letters of W = 1 must be below 256 (acb_utf8_write_device's caller checks) */
template <int W>
__global__ void __launch_bounds__(kCmpThreads) acb_utf8_write_kernel(const __grid_constant__ U8Args a, uint8_t *out, long long *out_off) {
    using T = std::conditional_t<W == 1, uint8_t, uint32_t>;
    __shared__ __align__(16) uint8_t s_buf[kCmpTile * W + 16];   /* the tile's letters */
    __shared__ long long s_off[kU8Stage];
    __shared__ long long s_range[2];
    for (long long h = (long long)blockIdx.x * blockDim.x + threadIdx.x; h <= a.n_hay; h += (long long)gridDim.x * blockDim.x)
        out_off[h] = a.loff[h] * W;
    const long long tile = blockIdx.x;
    if (tile >= a.n_tiles) return;
    const long long t0 = tile * kCmpTile, p0 = t0 + (long long)threadIdx.x * 32;
    long long lo = 0, hi = 0;
    const U8Offs o = u8_stage(a, t0, s_off, s_range, &lo, &hi);
    uint32_t w[10];
    u8_load(a.in, a.total, p0, w);
    const int valid = (int)max(min(32LL, a.total - p0), 0LL);
    T *dst = reinterpret_cast<T *>(s_buf) + a.gpre[tile * kCmpThreads + threadIdx.x];
    if (u8_ascii(w)) {
#pragma unroll
        for (int j = 0; j < 32; j++)
            if (j < valid) dst[j] = (T)u8_at(w, j);
    } else {
        const unsigned long long bnd = u8_bounds(a, o, lo, hi, p0);
        const uint32_t keep = u8_starts(w, bnd, valid);
        int n = 0;
#pragma unroll
        for (int j = 0; j < 32; j++) {
            if (!((keep >> j) & 1)) continue;
            uint32_t cp;
            u8_prefix(w, j, bnd, &cp);
            dst[n++] = (T)cp;
        }
    }
    __syncthreads();
    /* coalesced stores: bytes up to a 16-byte boundary of the destination, then 16-byte words, then the rest */
    const long long first = a.tile_pre[tile];
    uint8_t *d = out + first * W;
    const int nb = (int)(a.tile_pre[tile + 1] - first) * W;
    const int head = min(nb, (int)((16 - (reinterpret_cast<uintptr_t>(d) & 15)) & 15)), nmid = (nb - head) >> 4;
    if ((int)threadIdx.x < head) d[threadIdx.x] = s_buf[threadIdx.x];
    const int sh = (head & 3) * 8;
    const uint32_t *sw = reinterpret_cast<const uint32_t *>(s_buf) + (head >> 2);
    for (int i = threadIdx.x; i < nmid; i += kCmpThreads) {
        const uint32_t *q = sw + 4 * i;                    /* unaligned by head bytes in shared memory: funnel shifts */
        const uint32_t a0 = q[0], a1 = q[1], a2 = q[2], a3 = q[3], a4 = q[4];
        reinterpret_cast<uint4 *>(d + head)[i] = make_uint4(__funnelshift_r(a0, a1, sh), __funnelshift_r(a1, a2, sh),
                                                            __funnelshift_r(a2, a3, sh), __funnelshift_r(a3, a4, sh));
    }
    for (int i = head + (nmid << 4) + threadIdx.x; i < nb; i += kCmpThreads) d[i] = s_buf[i];
}

/* UTF-8 bytes of letter c: code points as Unicode encodes them (surrogates at 3 bytes, as "surrogatepass" does);
 * letters from 0x110000 up become U+FFFD */
__device__ __forceinline__ int u8_len(uint32_t c) { return c < 0x80u ? 1 : c < 0x800u ? 2 : c < 0x10000u ? 3 : c < 0x110000u ? 4 : 3; }

template <int W>
__device__ __forceinline__ uint32_t u8_letter(const uint8_t *in, long long i) {
    return W == 1 ? (uint32_t)in[i] : reinterpret_cast<const uint32_t *>(in)[i];
}

/* encode, count pass: out_off[h] = UTF-8 bytes of haystack h (one CTA per haystack, grid-stride), out_off[n_hay] = 0 */
template <int W>
__global__ void __launch_bounds__(256) acb_utf8_count_kernel(const uint8_t *in, const long long *off, long long n_hay, long long *out_off) {
    __shared__ unsigned long long s_sum;
    for (long long h = blockIdx.x; h < n_hay; h += gridDim.x) {
        if (threadIdx.x == 0) s_sum = 0;
        __syncthreads();
        const long long e = __ldg(off + h + 1) / W;
        unsigned int sum = 0;                              /* < 2^26: at most 2^31 letters of 4 bytes over 256 threads */
        for (long long i = __ldg(off + h) / W + threadIdx.x; i < e; i += 256) sum += u8_len(u8_letter<W>(in, i));
        sum = __reduce_add_sync(kFull, sum);
        if ((threadIdx.x & 31) == 0 && sum) atomicAdd(&s_sum, (unsigned long long)sum);
        __syncthreads();
        if (threadIdx.x == 0) out_off[h] = (long long)s_sum;
        __syncthreads();                                   /* s_sum is set again */
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) out_off[n_hay] = 0;
}

/* encode, write pass: the UTF-8 bytes of each haystack at out + out_off[h], when the total fits out_cap */
template <int W>
__global__ void __launch_bounds__(256) acb_utf8_encode_kernel(const uint8_t *in, const long long *off, long long n_hay,
                                                              const long long *out_off, uint8_t *out, long long out_cap) {
    using Scan = cub::BlockScan<int, 256>;
    __shared__ typename Scan::TempStorage tmp;
    if (out_off[n_hay] > out_cap) return;
    for (long long h = blockIdx.x; h < n_hay; h += gridDim.x) {
        long long base = out_off[h];
        const long long e = __ldg(off + h + 1) / W;
        for (long long c0 = __ldg(off + h) / W; c0 < e; c0 += 256) {
            const long long i = c0 + threadIdx.x;
            uint32_t c = i < e ? u8_letter<W>(in, i) : 0;
            if (c >= 0x110000u) c = 0xFFFDu;
            const int len = i < e ? u8_len(c) : 0;
            int pre, agg;
            Scan(tmp).ExclusiveSum(len, pre, agg);
            uint8_t *d = out + base + pre;
            if (len == 1) {
                d[0] = (uint8_t)c;
            } else if (len == 2) {
                d[0] = (uint8_t)(0xC0u | c >> 6); d[1] = (uint8_t)(0x80u | (c & 0x3Fu));
            } else if (len == 3) {
                d[0] = (uint8_t)(0xE0u | c >> 12); d[1] = (uint8_t)(0x80u | ((c >> 6) & 0x3Fu)); d[2] = (uint8_t)(0x80u | (c & 0x3Fu));
            } else if (len == 4) {
                d[0] = (uint8_t)(0xF0u | c >> 18); d[1] = (uint8_t)(0x80u | ((c >> 12) & 0x3Fu));
                d[2] = (uint8_t)(0x80u | ((c >> 6) & 0x3Fu)); d[3] = (uint8_t)(0x80u | (c & 0x3Fu));
            }
            base += agg;
            __syncthreads();                               /* tmp is used again */
        }
    }
}

thread_local float g_u8_ms[3] = {};                        /* kernel timing: decode pass 1, pass 2, encode */

/* the workspace of acb_utf8_decode_device, carved in this order */
struct U8Work {
    long long n_tiles;
    size_t bytes;
    U8Work(int64_t total, int64_t n_hay) {
        n_tiles = (total + kCmpTile - 1) / kCmpTile;
        const size_t groups = (size_t)n_tiles * kCmpThreads;
        auto up = [](size_t b) { return (b + 255) & ~(size_t)255; };
        bytes = up(groups * 4) + up(groups * 2) + up(((size_t)n_tiles + 1) * 8) + up((size_t)n_tiles * 8) + up(4) + up(8) +
                up(((size_t)n_hay + 1) * 8);
    }
    void carve_into(void *work, U8Args &a) const {
        char *p = static_cast<char *>(work);
        const size_t groups = (size_t)n_tiles * kCmpThreads;
        a.mask = carve<uint32_t>(p, groups);
        a.gpre = carve<uint16_t>(p, groups);
        a.tile_pre = carve<long long>(p, (size_t)n_tiles + 1);
        a.status = carve<unsigned long long>(p, (size_t)n_tiles);
        a.ctr = carve<unsigned int>(p, 1);
        a.err = carve<unsigned long long>(p, 1);
        a.loff = reinterpret_cast<long long *>(p);
        a.n_tiles = n_tiles;
    }
};

/* cub's scratch for the encode's exclusive sum over n_hay + 1 offsets */
static int u8_scan_bytes(int64_t n_hay, size_t *temp) {
    *temp = 0;
    CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, *temp, (long long *)nullptr, (long long *)nullptr, (int)(n_hay + 1)));
    return ACB_OK;
}

/* f() launched on s; with kernel timing on, *ms is its time from events made for this call (the call waits for them) */
template <class F>
static int u8_timed(cudaStream_t s, float *ms, F &&f) {
    if (!g_timing.load()) return f();
    cudaEvent_t e[2] = {nullptr, nullptr};
    int rc = ACB_OK;
    if (cudaEventCreate(&e[0]) != cudaSuccess || cudaEventCreate(&e[1]) != cudaSuccess || cudaEventRecord(e[0], s) != cudaSuccess) {
        acb_set_error("kernel timing events failed");
        rc = ACB_ECUDA;
    } else if ((rc = f()) == ACB_OK && (cudaEventRecord(e[1], s) != cudaSuccess || cudaEventSynchronize(e[1]) != cudaSuccess ||
                                        cudaEventElapsedTime(ms, e[0], e[1]) != cudaSuccess)) {
        acb_set_error("kernel timing events failed");
        rc = ACB_ECUDA;
    }
    for (cudaEvent_t ev : e) if (ev) cudaEventDestroy(ev);
    return rc;
}

/* the checks shared by the decode passes: batch shape, buffers, device */
static int u8_check(int device, const uint8_t *d_in, int64_t total_bytes, const int64_t *d_offsets, int64_t n_hay, int64_t stride_bytes,
                    const void *d_work, int64_t work_bytes) {
    if (total_bytes < 0 || n_hay < 0 || (total_bytes && !d_in) || work_bytes < 0) { acb_set_error("bad argument"); return ACB_EINVAL; }
    if (n_hay > 0x7fffffffLL) { acb_set_error("more than 2^31-1 haystacks in one batch"); return ACB_ERANGE; }
    if (!d_offsets) {
        int rc = check_stride(1, total_bytes, n_hay, stride_bytes, 0);
        if (rc != ACB_OK) return rc;
    }
    const U8Work wk(total_bytes, n_hay);
    if (wk.n_tiles > 0x7fffffffLL) { acb_set_error("batch too large to decode in one launch"); return ACB_ERANGE; }
    if ((int64_t)wk.bytes > work_bytes || !d_work) {
        acb_set_error("workspace of %lld bytes at %p, the batch needs %lld (acb_utf8_work_bytes)", (long long)work_bytes, d_work,
                      (long long)wk.bytes);
        return ACB_EINVAL;
    }
    if (reinterpret_cast<uintptr_t>(d_in) & 15) { acb_set_error("d_in must be 16-byte aligned"); return ACB_EINVAL; }
    CUDA_TRY(cudaSetDevice(device));
    return ACB_OK;
}

static void u8_args(U8Args &a, const uint8_t *d_in, int64_t total_bytes, const int64_t *d_offsets, int64_t n_hay, int64_t stride_bytes,
                    const void *d_work, int64_t *d_info, int strict) {
    a = U8Args{};
    a.in = d_in; a.total = total_bytes; a.off = reinterpret_cast<const long long *>(d_offsets); a.stride = stride_bytes; a.n_hay = n_hay;
    a.info = reinterpret_cast<long long *>(d_info);
    a.strict = strict;
    U8Work(total_bytes, n_hay).carve_into(const_cast<void *>(d_work), a);
}
} // namespace

extern "C" int acb_utf8_work_bytes(int64_t total_bytes, int64_t n_hay, int64_t *bytes) {
    if (!bytes || total_bytes < 0 || n_hay < 0) { acb_set_error("bad argument"); return ACB_EINVAL; }
    if (n_hay > 0x7fffffffLL - 1) { acb_set_error("more than 2^31-2 haystacks in one batch"); return ACB_ERANGE; }
    size_t temp = 0;
    if (int rc = u8_scan_bytes(n_hay, &temp)) return rc;
    *bytes = (int64_t)std::max(U8Work(total_bytes, n_hay).bytes, temp + 256);
    return ACB_OK;
}

extern "C" int acb_utf8_decode_device(int device, const uint8_t *d_in, int64_t total_bytes, const int64_t *d_offsets, int64_t n_hay,
                                      int64_t stride_bytes, int errors, void *d_work, int64_t work_bytes, int64_t *d_info, void *stream) {
    DeviceRestore keep_device;
    if (!d_info || (errors != ACB_UTF8_STRICT && errors != ACB_UTF8_REPLACE)) { acb_set_error("bad argument"); return ACB_EINVAL; }
    int rc = u8_check(device, d_in, total_bytes, d_offsets, n_hay, stride_bytes, d_work, work_bytes);
    if (rc) return rc;
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    U8Args a;
    u8_args(a, d_in, total_bytes, d_offsets, n_hay, stride_bytes, d_work, d_info, errors == ACB_UTF8_STRICT);
    g_u8_ms[0] = 0.f;
    CUDA_TRY(cudaMemsetAsync(d_info, 0, 5 * sizeof(int64_t), s));
    CUDA_TRY(cudaMemsetAsync(a.err, 0xff, sizeof(unsigned long long), s));
    CUDA_TRY(cudaMemsetAsync(a.ctr, 0, sizeof(unsigned int), s));
    CUDA_TRY(cudaMemsetAsync(a.tile_pre, 0, ((size_t)a.n_tiles + 1) * sizeof(long long), s));
    if (a.n_tiles) CUDA_TRY(cudaMemsetAsync(a.status, 0, (size_t)a.n_tiles * sizeof(unsigned long long), s));
    const CompactMeta meta{a.mask, a.gpre, a.tile_pre, a.n_tiles};
    return u8_timed(s, &g_u8_ms[0], [&]() -> int {
        int r;
        if (a.n_tiles) {
            acb_utf8_decode_kernel<<<(unsigned)a.n_tiles, kCmpThreads, 0, s>>>(a);
            if ((r = launched("UTF-8 decode"))) return r;
        }
        acb_utf8_offsets_kernel<<<(unsigned)((n_hay + 1 + 255) / 256), 256, 0, s>>>(meta, a);
        return launched("UTF-8 offsets");
    });
}

extern "C" int acb_utf8_write_device(int device, const uint8_t *d_in, int64_t total_bytes, const int64_t *d_offsets, int64_t n_hay,
                                     int64_t stride_bytes, const void *d_work, int64_t work_bytes, int width, uint8_t *d_out,
                                     int64_t *d_out_offsets, void *stream) {
    DeviceRestore keep_device;
    if ((width != 1 && width != 4) || !d_out_offsets || (total_bytes && !d_out)) { acb_set_error("bad argument"); return ACB_EINVAL; }
    int rc = u8_check(device, d_in, total_bytes, d_offsets, n_hay, stride_bytes, d_work, work_bytes);
    if (rc) return rc;
    if (reinterpret_cast<uintptr_t>(d_out) & 15) { acb_set_error("d_out must be 16-byte aligned"); return ACB_EINVAL; }
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    U8Args a;
    u8_args(a, d_in, total_bytes, d_offsets, n_hay, stride_bytes, d_work, nullptr, 0);
    g_u8_ms[1] = 0.f;
    const unsigned grid = (unsigned)std::max<long long>(a.n_tiles, 1);
    return u8_timed(s, &g_u8_ms[1], [&]() -> int {
        auto *oo = reinterpret_cast<long long *>(d_out_offsets);
        if (width == 1) acb_utf8_write_kernel<1><<<grid, kCmpThreads, 0, s>>>(a, d_out, oo);
        else acb_utf8_write_kernel<4><<<grid, kCmpThreads, 0, s>>>(a, d_out, oo);
        return launched("UTF-8 write");
    });
}

extern "C" int acb_utf8_encode_device(int device, const uint8_t *d_in, int64_t total_bytes, const int64_t *d_offsets, int64_t n_hay,
                                      int width, void *d_work, int64_t work_bytes, uint8_t *d_out, int64_t out_cap,
                                      int64_t *d_out_offsets, int64_t *d_total, void *stream) {
    DeviceRestore keep_device;
    if ((width != 1 && width != 4) || total_bytes < 0 || n_hay < 0 || (total_bytes && !d_in) || !d_offsets || !d_out_offsets ||
        !d_total || out_cap < 0 || (out_cap && !d_out) || work_bytes < 0) {
        acb_set_error("bad argument");
        return ACB_EINVAL;
    }
    if (n_hay > 0x7fffffffLL - 1) { acb_set_error("more than 2^31-2 haystacks in one batch"); return ACB_ERANGE; }
    size_t temp = 0;
    int rc = u8_scan_bytes(n_hay, &temp);
    if (rc) return rc;
    if ((int64_t)temp > work_bytes || (temp && !d_work)) {
        acb_set_error("workspace of %lld bytes at %p, the encode needs %lld (acb_utf8_work_bytes)", (long long)work_bytes, d_work, (long long)temp);
        return ACB_EINVAL;
    }
    CUDA_TRY(cudaSetDevice(device));
    int sms = 0;
    CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    auto *off = reinterpret_cast<const long long *>(d_offsets);
    auto *oo = reinterpret_cast<long long *>(d_out_offsets);
    const unsigned grid = (unsigned)std::max<long long>(std::min<long long>(n_hay, (long long)sms * 16), 1);
    g_u8_ms[2] = 0.f;
    return u8_timed(s, &g_u8_ms[2], [&]() -> int {
        int r;
        if (width == 1) acb_utf8_count_kernel<1><<<grid, 256, 0, s>>>(d_in, off, n_hay, oo);
        else acb_utf8_count_kernel<4><<<grid, 256, 0, s>>>(d_in, off, n_hay, oo);
        if ((r = launched("UTF-8 count"))) return r;
        CUDA_TRY(cub::DeviceScan::ExclusiveSum(d_work, temp, oo, oo, (int)(n_hay + 1), s));
        CUDA_TRY(cudaMemcpyAsync(d_total, oo + n_hay, sizeof(int64_t), cudaMemcpyDeviceToDevice, s));
        if (!out_cap) return ACB_OK;
        if (width == 1) acb_utf8_encode_kernel<1><<<grid, 256, 0, s>>>(d_in, off, n_hay, oo, d_out, out_cap);
        else acb_utf8_encode_kernel<4><<<grid, 256, 0, s>>>(d_in, off, n_hay, oo, d_out, out_cap);
        return launched("UTF-8 encode");
    });
}

extern "C" int acb_last_utf8_ms(float *ms, int32_t n) {
    if (!ms || n < 0 || n > 3) { acb_set_error("bad argument"); return ACB_EINVAL; }
    for (int i = 0; i < n; i++) ms[i] = g_u8_ms[i];
    return ACB_OK;
}

/* ------------------------------------------------------------ UTF-8 stream carries (DESIGN section 4.21) */
/* Per stream, the bytes of an unfinished letter that a UTF-8 stream holds back from one feed to the next, in one 32-bit
 * word: bytes 0..2 the held bytes, byte 3 their number (0..3).  A stage builds, per chunk h of stream s, carry_s ||
 * chunk_h without its new held tail into a ragged batch the UTF-8 decode takes as it is, and stages the new tail in a
 * second word per chunk; a commit copies the staged words to the streams.  The held tail is the one CPython's
 * incremental decoder keeps: the bytes from the last non-continuation byte among the last 3 to the end, when that
 * byte's maximal valid prefix (u8_prefix's rule) runs to the end and is shorter than its sequence, and also ED A0-BF,
 * which CPython keeps until a third byte arrives. */
namespace {
constexpr int kU8cTile = 4096;                             /* staged bytes per block turn of the gather */
constexpr int kU8cHays = 512;                              /* staged offsets a gather block keeps in shared memory */

struct U8cArgs {
    const uint8_t *in; long long total; const long long *off; long long stride; long long n;   /* the caller's chunks */
    const int32_t *ids; long long n_streams;
    const uint32_t *carry; uint32_t *next;                 /* per stream; per chunk */
    long long *soff;                                       /* staged byte offsets [n + 1] */
    uint8_t *staged; long long span;                       /* staged bytes, zero from soff[n] to span */
    int final;
};

__device__ __forceinline__ long long u8c_stream(const U8cArgs &a, long long h) {
    const long long s = a.ids ? (long long)__ldg(a.ids + h) : h;
    return (s >= 0 && s < a.n_streams) ? s : -1;
}

/* the held tail of a text whose last m (<= 3) bytes are bytes 0..m-1 of v */
__device__ __forceinline__ int u8c_hold(uint32_t v, int m) {
    for (int p = m - 1; p >= 0; --p) {
        const uint32_t b0 = (v >> (8 * p)) & 255u;
        if ((b0 & 0xC0u) == 0x80u) continue;
        const int d = m - p, need = b0 < 0xC2u ? 0 : b0 < 0xE0u ? 2 : b0 < 0xF0u ? 3 : b0 < 0xF5u ? 4 : 0;
        if (d >= need) return 0;
        const uint32_t b1 = (v >> (8 * (p + 1))) & 255u;   /* the bytes after b0 are continuation bytes */
        /* as u8_prefix, except that ED A0-BF is held: CPython's decoder waits for a third byte before it calls it invalid */
        const uint32_t lo = b0 == 0xE0u ? 0xA0u : b0 == 0xF0u ? 0x90u : 0x80u, hi = b0 == 0xF4u ? 0x8Fu : 0xBFu;
        return d == 1 || (b1 >= lo && b1 <= hi) ? d : 0;
    }
    return 0;
}

/* next[h] = the new held tail of chunk h's stream; soff[h] = bytes of carry || chunk without it (soff[n] = 0), for the
 * exclusive scan that makes them offsets */
__global__ void acb_u8c_len_kernel(const __grid_constant__ U8cArgs a) {
    for (long long h = (long long)blockIdx.x * blockDim.x + threadIdx.x; h <= a.n; h += (long long)gridDim.x * blockDim.x) {
        if (h == a.n) { a.soff[h] = 0; continue; }
        const long long s = u8c_stream(a, h);
        const uint32_t c = s < 0 ? 0u : a.carry[s];
        const int cl = (int)(c >> 24);
        const long long b0 = hay_start(a.off, a.stride, h), len = cl + hay_start(a.off, a.stride, h + 1) - b0;
        const int m = (int)min(len, 3LL);
        uint32_t v = 0;                                    /* the last m bytes of carry || chunk */
        for (int j = 0; j < m; j++) {
            const long long i = len - m + j;
            v |= (i < cl ? (c >> (8 * i)) & 255u : (uint32_t)__ldg(a.in + b0 + i - cl)) << (8 * j);
        }
        const int k = a.final ? 0 : u8c_hold(v, m);
        a.next[h] = (uint32_t)k << 24 | (k ? v >> (8 * (m - k)) : 0u);
        a.soff[h] = len - k;
    }
}

/* last j in [lo, hi] with o(j) <= x, o(lo) <= x */
template <class O>
__device__ __forceinline__ long long u8c_find(const O &o, long long lo, long long hi, long long x) {
    while (lo < hi) {
        const long long mid = (lo + hi + 1) >> 1;
        if (o(mid) <= x) lo = mid; else hi = mid - 1;
    }
    return lo;
}

/* The ragged gather: staged haystack h = [soff[h], soff[h+1]) is its stream's carried bytes, then its chunk, up to its
 * length; bytes from soff[n] to span are zero.  Blocks take tiles of kU8cTile staged bytes, start at the tile's first
 * haystack ts[t] (acb_sl_tiles_kernel) and keep the following offsets in shared memory; each thread writes one 16-byte
 * block, from two aligned 16-byte loads (rp_load16) when it lies in one chunk's bytes, else byte by byte. */
static_assert(kU8cTile == kSlTile, "the gather's tiles are those acb_sl_tiles_kernel finds");
__global__ void __launch_bounds__(256) acb_u8c_gather_kernel(const __grid_constant__ U8cArgs a, const long long *ts) {
    __shared__ long long s_off[kU8cHays + 1];
    const long long n_tiles = (a.span + kU8cTile - 1) / kU8cTile, total = __ldg(a.soff + a.n);
    for (long long t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        const long long c0 = t * kU8cTile, h0 = a.n ? __ldg(ts + t) : 0;
        __syncthreads();                                   /* the previous tile's readers are done */
        const int nh = (int)min((long long)kU8cHays, a.n - h0);
        for (int j = threadIdx.x; j <= nh; j += blockDim.x) s_off[j] = __ldg(a.soff + h0 + j);
        __syncthreads();
        const long long c = c0 + (long long)threadIdx.x * 16;
        if (c >= a.span) continue;
        if (c >= total) {                                  /* the zeros after the last haystack */
            if (c + 16 <= a.span) *reinterpret_cast<uint4 *>(a.staged + c) = make_uint4(0u, 0u, 0u, 0u);
            else for (long long o = c; o < a.span; o++) a.staged[o] = 0;
            continue;
        }
        const auto O = [&](long long j) { return j - h0 <= nh ? s_off[j - h0] : __ldg(a.soff + j); };
        const auto F = [&](long long from, long long x) { return u8c_find(O, from, x < s_off[nh] ? h0 + nh - 1 : a.n - 1, x); };
        long long h = F(h0, c), lo = O(h), hi = O(h + 1), src = 0;
        uint32_t cw = 0;                                   /* the carry of haystack h's stream */
        const auto enter = [&]() {
            const long long s = u8c_stream(a, h);
            cw = s < 0 ? 0u : a.carry[s];
            src = hay_start(a.off, a.stride, h) - (long long)(cw >> 24);   /* chunk byte of staged byte lo, less the carry */
        };
        enter();
        if (c - lo >= (long long)(cw >> 24) && c + 16 <= hi) {
            *reinterpret_cast<uint4 *>(a.staged + c) = rp_load16(a.in, src + (c - lo));
            continue;
        }
        uint32_t w[4] = {0u, 0u, 0u, 0u};
#pragma unroll
        for (int j = 0; j < 16; j++) {
            const long long o = c + j;
            if (o < total) {
                if (o >= hi) { h = F(h + 1, o); lo = O(h); hi = O(h + 1); enter(); }
                const long long rel = o - lo;
                const uint32_t b = rel < (long long)(cw >> 24) ? (cw >> (8 * rel)) & 255u : (uint32_t)__ldg(a.in + src + rel);
                w[j >> 2] |= b << (8 * (j & 3));
            }
        }
        if (c + 16 <= a.span) {
            *reinterpret_cast<uint4 *>(a.staged + c) = make_uint4(w[0], w[1], w[2], w[3]);
        } else {
#pragma unroll
            for (int j = 0; j < 16; j++)
                if (c + j < a.span) a.staged[c + j] = (uint8_t)(w[j >> 2] >> (8 * (j & 3)));
        }
    }
}

/* carry[stream of chunk h] = next[h] */
__global__ void acb_u8c_commit_kernel(const int32_t *ids, long long n, long long n_streams, const uint32_t *next, uint32_t *carry) {
    for (long long h = (long long)blockIdx.x * blockDim.x + threadIdx.x; h < n; h += (long long)gridDim.x * blockDim.x) {
        const long long s = ids ? (long long)__ldg(ids + h) : h;
        if (s >= 0 && s < n_streams) carry[s] = next[h];
    }
}

/* carry[ids[i]] = 0 */
__global__ void acb_u8c_clear_kernel(const int32_t *ids, long long n, long long n_streams, uint32_t *carry) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const long long s = ids[i];
        if (s >= 0 && s < n_streams) carry[s] = 0u;
    }
}
} // namespace

struct acb_utf8_carry {
    int device = 0;
    int sm_count = 1;
    long long n = 0;
    uint32_t *d_carry = nullptr;                           /* [n]: the committed tails */
    uint32_t *d_next = nullptr;                            /* [n]: the tails the last stage made, per chunk */
    long long staged = -1;                                 /* chunks of the last stage, -1 after a commit */
    long long *d_ts = nullptr; size_t ts_cap = 0;          /* the first staged haystack of every gather tile */
    int32_t *d_ids = nullptr; size_t ids_cap = 0;          /* the ids of a reset */
    uint8_t *d_tmp = nullptr; size_t tmp_cap = 0;          /* cub scratch */
};

/* a grid-stride launch over `items`: a block per 256, at most 16 per SM */
static unsigned u8c_blocks(const acb_utf8_carry *c, long long items) {
    return (unsigned)std::max<long long>(std::min<long long>((items + 255) / 256, (long long)c->sm_count * 16), 1);
}

extern "C" void acb_utf8_carry_free(acb_utf8_carry *c) {
    DeviceRestore keep_device;
    if (!c) return;
    cudaSetDevice(c->device);
    cudaFree(c->d_carry); cudaFree(c->d_next); cudaFree(c->d_ids); cudaFree(c->d_tmp); cudaFree(c->d_ts);
    delete c;
}

extern "C" int acb_utf8_carry_new(int device, int64_t n_streams, acb_utf8_carry **out) {
    DeviceRestore keep_device;
    if (!out || n_streams < 0) { acb_set_error("bad argument"); return ACB_EINVAL; }
    *out = nullptr;
    if (n_streams > 0x7fffffffLL) { acb_set_error("more than 2^31-1 streams"); return ACB_ERANGE; }
    CUDA_TRY(cudaSetDevice(device));
    acb_utf8_carry *c = new (std::nothrow) acb_utf8_carry();
    if (!c) { acb_set_error("out of memory"); return ACB_ENOMEM; }
    c->device = device;
    c->n = n_streams;
    const size_t n = (size_t)std::max<int64_t>(n_streams, 1);
    cudaError_t e = cudaDeviceGetAttribute(&c->sm_count, cudaDevAttrMultiProcessorCount, device);
    if (e == cudaSuccess) e = cudaMalloc(reinterpret_cast<void **>(&c->d_carry), n * sizeof(uint32_t));
    if (e == cudaSuccess) e = cudaMemset(c->d_carry, 0, n * sizeof(uint32_t));
    if (e == cudaSuccess) e = cudaMalloc(reinterpret_cast<void **>(&c->d_next), n * sizeof(uint32_t));
    if (e != cudaSuccess) {
        acb_set_error("allocating the carries of %lld streams: %s", (long long)n_streams, cudaGetErrorString(e));
        acb_utf8_carry_free(c);
        return ACB_ECUDA;
    }
    *out = c;
    return ACB_OK;
}

extern "C" int acb_utf8_carry_reset(acb_utf8_carry *c, const int32_t *ids, int64_t n) {
    DeviceRestore keep_device;
    if (!c || n < 0 || (n && !ids)) { acb_set_error("bad argument"); return ACB_EINVAL; }
    for (int64_t i = 0; ids && i < n; i++)
        if (ids[i] < 0 || ids[i] >= c->n) { acb_set_error("stream id %d out of range [0, %lld)", ids[i], c->n); return ACB_EINVAL; }
    CUDA_TRY(cudaSetDevice(c->device));
    if (!ids) {
        CUDA_TRY(cudaMemset(c->d_carry, 0, (size_t)std::max<long long>(c->n, 1) * sizeof(uint32_t)));
        return ACB_OK;
    }
    if (n == 0) return ACB_OK;
    int rc = ensure(&c->d_ids, &c->ids_cap, (size_t)n);
    if (rc) return rc;
    CUDA_TRY(cudaMemcpy(c->d_ids, ids, (size_t)n * sizeof(int32_t), cudaMemcpyHostToDevice));
    acb_u8c_clear_kernel<<<u8c_blocks(c, n), 256>>>(c->d_ids, n, c->n, c->d_carry);
    if ((rc = launched("UTF-8 carry reset"))) return rc;
    CUDA_TRY(cudaDeviceSynchronize());
    return ACB_OK;
}

extern "C" int acb_utf8_carry_pending(acb_utf8_carry *c, int64_t *out, int64_t cap) {
    DeviceRestore keep_device;
    if (!c || cap < c->n || (c->n && !out)) { acb_set_error("bad argument"); return ACB_EINVAL; }
    if (!c->n) return ACB_OK;
    CUDA_TRY(cudaSetDevice(c->device));
    std::vector<uint32_t> w;
    try { w.resize((size_t)c->n); } catch (const std::exception &) { acb_set_error("out of host memory"); return ACB_ENOMEM; }
    CUDA_TRY(cudaMemcpy(w.data(), c->d_carry, (size_t)c->n * sizeof(uint32_t), cudaMemcpyDeviceToHost));
    for (long long s = 0; s < c->n; s++) out[s] = (int64_t)(w[s] >> 24);
    return ACB_OK;
}

extern "C" int acb_utf8_carry_bytes(acb_utf8_carry *c, int32_t id, uint8_t *out, int32_t *n) {
    DeviceRestore keep_device;
    if (!c || !out || !n || id < 0 || id >= c->n) { acb_set_error("bad argument"); return ACB_EINVAL; }
    CUDA_TRY(cudaSetDevice(c->device));
    uint32_t w = 0;
    CUDA_TRY(cudaMemcpy(&w, c->d_carry + id, sizeof(w), cudaMemcpyDeviceToHost));
    *n = (int32_t)(w >> 24);
    for (int j = 0; j < 3; j++) out[j] = (uint8_t)(w >> (8 * j));
    return ACB_OK;
}

extern "C" int acb_utf8_carry_stage_device(acb_utf8_carry *c, const uint8_t *d_chunks, int64_t total_bytes, const int64_t *d_offsets,
                                           int64_t n_chunks, int64_t stride_bytes, const int32_t *d_ids, int final, uint8_t *d_staged,
                                           int64_t staged_cap, int64_t *d_staged_offsets, void *stream) {
    DeviceRestore keep_device;
    if (!c || total_bytes < 0 || n_chunks < 0 || (total_bytes && !d_chunks) || !d_staged_offsets || staged_cap < 0) {
        acb_set_error("bad argument");
        return ACB_EINVAL;
    }
    if (n_chunks > 0x7fffffffLL - 1) { acb_set_error("more than 2^31-2 chunks in one feed"); return ACB_ERANGE; }
    if (n_chunks > c->n) { acb_set_error("%lld chunks for %lld streams", (long long)n_chunks, c->n); return ACB_EINVAL; }
    if (!d_offsets) {
        int rc = check_stride(1, total_bytes, n_chunks, stride_bytes, 0);
        if (rc != ACB_OK) return rc;
    }
    const long long span = total_bytes + 3 * n_chunks;
    if (staged_cap < span || (span && !d_staged)) {
        acb_set_error("staged buffer of %lld bytes, the feed needs %lld (total_bytes + 3 * n_chunks)", (long long)staged_cap, span);
        return ACB_EINVAL;
    }
    if ((reinterpret_cast<uintptr_t>(d_staged) | reinterpret_cast<uintptr_t>(d_chunks)) & 15) {
        acb_set_error("d_chunks and d_staged must be 16-byte aligned");
        return ACB_EINVAL;
    }
    CUDA_TRY(cudaSetDevice(c->device));
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    U8cArgs a;
    memset(&a, 0, sizeof(a));
    a.in = d_chunks; a.total = total_bytes; a.off = reinterpret_cast<const long long *>(d_offsets); a.stride = stride_bytes; a.n = n_chunks;
    a.ids = d_ids; a.n_streams = c->n; a.carry = c->d_carry; a.next = c->d_next;
    a.soff = reinterpret_cast<long long *>(d_staged_offsets); a.staged = d_staged; a.span = span; a.final = final ? 1 : 0;
    acb_u8c_len_kernel<<<u8c_blocks(c, n_chunks + 1), 256, 0, s>>>(a);
    int rc = launched("UTF-8 carry lengths");
    if (rc) return rc;
    size_t temp = 0;
    CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, temp, a.soff, a.soff, (int)(n_chunks + 1), s));
    if ((rc = ensure(&c->d_tmp, &c->tmp_cap, temp))) return rc;
    temp = c->tmp_cap;
    CUDA_TRY(cub::DeviceScan::ExclusiveSum(c->d_tmp, temp, a.soff, a.soff, (int)(n_chunks + 1), s));
    if (span) {
        const long long n_tiles = (span + kU8cTile - 1) / kU8cTile;
        if ((rc = ensure(&c->d_ts, &c->ts_cap, (size_t)n_tiles))) return rc;
        if (n_chunks) {
            acb_sl_tiles_kernel<<<u8c_blocks(c, n_tiles), 256, 0, s>>>(a.soff, n_chunks, span, c->d_ts);
            if ((rc = launched("UTF-8 carry gather tiles"))) return rc;
        }
        acb_u8c_gather_kernel<<<(unsigned)std::min<long long>(n_tiles, (long long)c->sm_count * 8), 256, 0, s>>>(a, c->d_ts);
        if ((rc = launched("UTF-8 carry gather"))) return rc;
    }
    c->staged = n_chunks;
    return ACB_OK;
}

extern "C" int acb_utf8_carry_commit_device(acb_utf8_carry *c, const int32_t *d_ids, int64_t n_chunks, void *stream) {
    DeviceRestore keep_device;
    if (!c || n_chunks < 0) { acb_set_error("bad argument"); return ACB_EINVAL; }
    if (n_chunks != c->staged) {
        acb_set_error("a commit of %lld chunks after a stage of %lld (-1: none since the last commit)", (long long)n_chunks, c->staged);
        return ACB_EINVAL;
    }
    CUDA_TRY(cudaSetDevice(c->device));
    c->staged = -1;
    if (n_chunks == 0) return ACB_OK;
    acb_u8c_commit_kernel<<<u8c_blocks(c, n_chunks), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(d_ids, n_chunks, c->n, c->d_next,
                                                                                                          c->d_carry);
    return launched("UTF-8 carry commit");
}
