/*
 * acb_device.cu -- sm_90a scan kernels and the device half of the C ABI (include/acb200.h).
 *
 * ACB_ALGO_FILTER (the fast path) is ONE launch per <= 2 GiB segment of the batch, of one of two streaming kernels
 * (both persistent, one CTA per SM, warp specialised):
 *
 *  acb_stream_kernel<NW,STRIDE,MODE>   SINGLE placements of the gram filter (any gram length and stride)
 *  acb_pair_kernel<L2B>                PAIR placement (gram 4, stride 1, 1-byte letters: one filter word per two positions)
 *      A producer warp claims 20 KiB tiles of the flat haystack buffer from an atomic counter and moves them
 *      into a 3-stage shared-memory ring with cp.async.bulk (the TMA engine) and mbarriers; the consumer warps take
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

#include <algorithm>
#include <atomic>
#include <mutex>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <exception>
#include <new>
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
    unsigned int n_tiles;          /* kTileBytes tiles in the segment */
    unsigned int *work_ctr;        /* [0] next tile, [1] CTAs done */
    uint2 *cand;                   /* candidate entries, kWarpCand per consumer warp of every CTA: {position in the segment, anchor tag} */
    int stride_shift;              /* log2(stride_bytes) when it is a power of two, else -1 */
    int letter_shift;              /* log2(L) */
};

/* ---------------------------------------------------------------- helpers */

/* aligned 32-bit word at byte offset a (a % 4 == 0), zero filled past the end of the buffer */
__device__ __forceinline__ uint32_t load_word(const uint8_t *hay, long long a, long long total) {
    if (a + 4 <= total) return __ldg(reinterpret_cast<const uint32_t *>(hay + a));
    uint32_t v = 0;
    for (int b = 0; b < 4; b++) if (a + b < total) v |= (uint32_t)hay[a + b] << (8 * b);
    return v;
}

__device__ __forceinline__ void find_haystack(const ScanParams &p, long long q, long long &h, long long &hs, long long &he) {
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
__device__ __forceinline__ void load_text(const ScanParams &p, long long x, uint32_t (&w)[6]) {
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
 * (cp.async.bulk + mbarrier); `stages` = offset of the ring in the CTA's shared memory. */
template <int NCONS>
__device__ __forceinline__ void stream_producer(const ScanParams &p, uint8_t *smem_raw, uint32_t sbase, uint32_t stages,
                                                uint32_t bar_full, uint32_t bar_empty, volatile uint32_t *s_tile, int lane) {
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
        stream_producer<kConsumers>(p, smem_raw, sbase, lay.stages, bar_full, bar_empty, s_tile, lane);
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
 * acb_pair_kernel: the stream kernel of the PAIR placement (gram 4, stride 1, 1-byte letters; acb_hash.h).  Same ring,
 * same producer, same dynamic slices; what differs is everything a consumer warp does with its slice:
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
static_assert((kPairConsumers + kTileSlices - 1) / kTileSlices + 2 < 2 * ACB_STAGES && kPairThreads <= 1024, "pair kernel shape");
constexpr int kPairRing = 64;                                /* candidate ring entries per consumer warp */
constexpr int kPairItems = 64;                               /* item list entries (uint16) per consumer warp */

struct PairSmem {
    uint32_t bitmap, bitmap2, stages, ring, items, bars, tiles, next, total;
};
__host__ __device__ inline PairSmem pair_smem(int log1, int log2b) {
    PairSmem s;
    uint32_t o = 0;
    s.bitmap = o;    o += 1u << (log1 - 3);                       /* >= 1 KiB: level 2 follows without a gap, as in bm1 */
    s.bitmap2 = o;   o += 1u << (log2b - 3);                      o = (o + 127u) & ~127u;
    s.stages = o;    o += (uint32_t)kStages * kStageBytes;
    s.ring = o;      o += (uint32_t)kPairConsumers * kPairRing * 8u;
    s.items = o;     o += (uint32_t)kPairConsumers * kPairItems * 2u;
    s.bars = o;      o += 2u * kStages * 8u;
    s.tiles = o;     o += (uint32_t)kStages * 4u;
    s.next = o;      o += 4u;
    s.total = (o + 15u) & ~15u;
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

/* one turn of a warp's candidates (ring entries head .. head + n - 1, n <= 32, one per lane) through the anchor table.
 * Not inlined: the streaming loop keeps its registers and its schedule, and this runs once per five slices or so. */
__device__ __noinline__ void pair_resolve(const ScanParams &p, uint32_t sring, unsigned int head, unsigned int n) {
    const int lane = threadIdx.x & 31;
    const uint32_t lt_mask = (1u << lane) - 1u;
    bool hit = false;
    int32_t rh = 0, re = 0, rk = 0;
    if ((unsigned)lane < n) {
        const uint32_t amask = (1u << p.logA) - 1u;
        const uint2 e = lds64(sring + (((head + (unsigned)lane) & (kPairRing - 1u)) << 3));
        const long long q = p.seg_begin + (long long)e.x;
        uint32_t tq[6];
        load_text(p, q, tq);
        uint32_t slot = e.y >> (32 - p.logA);
        uint4 e0 = __ldg(p.anchors + 2 * (size_t)slot), e1 = __ldg(p.anchors + 2 * (size_t)slot + 1);
        while (e0.x != 0u && e0.x != e.y) {                      /* a foreign tag in the way: linear probing */
            slot = (slot + 1) & amask;
            e0 = __ldg(p.anchors + 2 * (size_t)slot);
            e1 = __ldg(p.anchors + 2 * (size_t)slot + 1);
        }
        if (e0.x != 0u) {
            if ((int32_t)e0.y >= 0 && (e0.z & 0x100ffu) == 0x10000u) {   /* the tag's ONE entry: UNIQUE, anchored at its first byte */
                const uint32_t kw[5] = {e0.w, e1.x, e1.y, e1.z, e1.w};
                const int len = (int)((e0.z >> 8) & 0xffu);
                long long h, hs, he;
                find_haystack(p, q, h, hs, he);
                hit = q + len <= he && text_equals(tq, q, len, kw);
                rh = (int32_t)h;
                re = (int32_t)(((q + len - hs) >> p.letter_shift) - 1);
                rk = (int32_t)e0.y;
            } else {
                pair_resolve_general(p, q, e.y, slot, e0, e1);
            }
        }
    }
    /* the hits of the warp: ONE atomicAdd on the record counter, records stored straight to the record buffer */
    const unsigned mh = __ballot_sync(kFull, hit);
    if (mh) {
        unsigned long long base = 0;
        if (lane == 0) base = atomicAdd(p.count, (unsigned long long)__popc(mh));
        base = __shfl_sync(kFull, base, 0) + (unsigned long long)__popc(mh & lt_mask);
        if (hit && base < (unsigned long long)p.cap) { acb_match m; m.hay_id = rh; m.end_index = re; m.key_id = rk; p.out[base] = m; }
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
    const uint32_t bar_full = sbase + lay.bars, bar_empty = bar_full + 8u * kStages;
    volatile uint32_t *s_tile = reinterpret_cast<volatile uint32_t *>(smem_raw + lay.tiles);

    if (tid == 0) {
        *reinterpret_cast<unsigned int *>(smem_raw + lay.next) = 0u;
        for (int s = 0; s < kStages; s++) {
            mbar_init(bar_full + 8u * s, 1);
            mbar_init(bar_empty + 8u * s, kTileSlices);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    const uint32_t seg_len = (uint32_t)(p.seg_end - p.seg_begin);        /* <= 2^31 */

    if (warp == kPairConsumers) {
        /* the producer starts at once: the first tiles are on their way while the consumers fetch the bitmap */
        stream_producer<kPairConsumers>(p, smem_raw, sbase, lay.stages, bar_full, bar_empty, s_tile, lane);
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
        const uint32_t lane5 = (uint32_t)lane << 5;
        unsigned int n_cand = 0, head = 0;                               /* warp-uniform: entries [head, head + n_cand) of the ring */

        for (;;) {
            unsigned int g = 0;
            if (lane == 0) asm volatile("atom.shared.add.u32 %0, [%1], 1;" : "=r"(g) : "r"(snext) : "memory");
            g = __shfl_sync(kFull, g, 0);
            const uint32_t fill = g / (uint32_t)kTileSlices, slice_off = (g % (uint32_t)kTileSlices) * (uint32_t)kSliceBytes;
            const uint32_t stage = fill % (uint32_t)kStages;
            mbar_wait(bar_full + 8u * stage, (fill / (uint32_t)kStages) & 1u);
            const uint32_t tile = s_tile[stage];
            if (tile == kNoTile) break;
            const uint32_t tile_off = tile * (uint32_t)kTileBytes;       /* relative to the segment */
            const uint32_t n_valid = (seg_len - tile_off < (uint32_t)kTileBytes) ? seg_len - tile_off : (uint32_t)kTileBytes;
            const uint32_t slice_saddr = sbase + lay.stages + stage * (uint32_t)kStageBytes + slice_off;
            const uint32_t pos_base = tile_off + slice_off;
            uint32_t pend = 0;       /* bit y < 16: position 16 * lane + y of the slice passed level 1; y >= 16: position 512 + 16 * lane + y - 16 */
            if (slice_off < n_valid) {                                   /* warp-uniform */
                const uint32_t saddr = slice_saddr + (uint32_t)lane * 16u;
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
            /* items: the pending positions of all lanes go to the list -- an exclusive scan of the lanes' counts places
               them (dense text, more than the list holds: ballot rounds, one position per lane and round, a pass at a
               time) -- and are worked off 32 at a time */
            unsigned int tot = __reduce_add_sync(kFull, (unsigned)__popc(pend));
            while (tot) {
                unsigned int n_items;
                if (tot <= (unsigned)kPairItems) {
                    const unsigned int cnt = (unsigned)__popc(pend);
                    unsigned int incl = cnt;
#pragma unroll
                    for (int d = 1; d < 32; d <<= 1) {
                        const unsigned int v = __shfl_up_sync(kFull, incl, d);
                        if (lane >= d) incl += v;
                    }
                    uint32_t at = sitems + 2u * (incl - cnt);
                    while (pend) {
                        const uint32_t z = (uint32_t)__clz((int)pend);
                        pend ^= 0x80000000u >> z;
                        sts16(at, lane5 | (z ^ 31u));                     /* lane << 5 | bit */
                        at += 2u;
                    }
                    n_items = tot;
                    tot = 0;
                } else {
                    n_items = 0;
                    do {
                        const unsigned int mp = __ballot_sync(kFull, pend != 0u);
                        if (pend) {
                            const uint32_t z = (uint32_t)__clz((int)pend);
                            pend ^= 0x80000000u >> z;
                            sts16(sitems + 2u * (n_items + (unsigned)__popc(mp & lt_mask)), lane5 | (z ^ 31u));
                        }
                        n_items += (unsigned)__popc(mp);
                    } while (n_items <= (unsigned)(kPairItems - 32));
                    tot -= n_items;
                }
                __syncwarp();
                for (unsigned int base = 0; base < n_items;) {
                    if (n_cand == (unsigned)kPairRing) {                /* one slice alone filled the ring */
                        __syncwarp();                                    /* the entries were written by other lanes */
                        pair_resolve(p, sring, head, 32u); head += 32u; n_cand -= 32u;
                        continue;
                    }
                    unsigned int take = n_items - base;
                    if (take > 32u) take = 32u;
                    if (take > (unsigned)kPairRing - n_cand) take = (unsigned)kPairRing - n_cand;
                    bool ok = false;
                    uint32_t pos = 0, tag = 0;
                    if ((unsigned)lane < take) {
                        const uint32_t it = lds16(sitems + 2u * (base + (unsigned)lane));
                        const uint32_t y = it & 31u;
                        const uint32_t t = ((it >> 1) & 0x1f0u) + ((y & 16u) * 31u + y);       /* 16 * lane + y, second run: + 496 */
                        const uint32_t ga = slice_saddr + t, wa = ga & ~3u;
                        const uint32_t lo = lds32(wa), hi = lds32(wa + 4u);
                        const uint32_t w = __funnelshift_r(lo, hi, ga << 3);                    /* wrap shift: (ga & 3) * 8 */
                        tag = (w * mul2) | 1u;
                        const uint32_t word = lds_bitmap((tag >> shy_w) * four + sbm2);
                        ok = (__funnelshift_r(word, 0u, tag >> shy_a) & __funnelshift_r(word, 0u, tag >> shy_b) & 1u) != 0u;
                        pos = pos_base + t;
                    }
                    if (p.log3) {                                        /* very large key sets: the tag bitmap in L2 as well */
                        const uint32_t i0 = (tag * ACB_TAGMAP_MIX) >> (32 - p.log3);
                        if (ok) ok = ((__ldg(p.bm3 + (i0 >> 5)) >> (i0 & 31u)) & 1u) != 0u;
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
                    base += take;
                }
                __syncwarp();
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
    int32_t state = (h == 0) ? p.long_init : 0, last_node = -1;     /* the walk of a stream goes on where the last chunk left it */
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
}

__global__ void acb_flag_goto_kernel(int32_t *gto, const int32_t *key_of, size_t n) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const int32_t v = gto[i];
        if (v >= 0 && key_of[v] >= 0) gto[i] = v | kTermBit;
    }
}

} // namespace

/* ------------------------------------------------------------- the table */

struct acb_table {
    int device = 0;
    int sm_count = 0;
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
    void *d_sort = nullptr; size_t sort_cap = 0;         /* radix-sort scratch */
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
    if (!tb) return;
    cudaSetDevice(tb->device);
    cudaFree(tb->d_lfail); cudaFree(tb->d_cls); cudaFree(tb->d_goto); cudaFree(tb->d_fail); cudaFree(tb->d_keyof);
    cudaFree(tb->d_outptr); cudaFree(tb->d_outidx); cudaFree(tb->d_keylen); cudaFree(tb->d_bm1); cudaFree(tb->d_bm3); cudaFree(tb->d_anchors);
    cudaFree(tb->d_sort); cudaFree(tb->d_work); cudaFree(tb->d_cand); cudaFree(tb->d_long_final); cudaFree(tb->w_hay); cudaFree(tb->w_off); cudaFree(tb->w_out); cudaFree(tb->w_count);
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
    delete tb;
}

extern "C" int acb_table_upload(const acb_trie *t, int device, acb_table **out) {
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
extern "C" int64_t acb_launch_count(void) { return g_launches.load(); }
extern "C" int acb_set_kernel_timing(int enabled) { g_timing.store(enabled ? 1 : 0); return ACB_OK; }
extern "C" float acb_last_kernel_ms(void) { return g_last_ms; }

/* ------------------------------------------------------------- launching */

constexpr int kMaxDevices = 64;                              /* opt-in caches below are per device */

template <int NW, int STRIDE, int MODE>
static int launch_stream_m(const ScanParams &p, int grid, cudaStream_t s) {
    auto kern = acb_stream_kernel<NW, STRIDE, MODE>;
    const size_t smem = stream_smem(p.log1).total;
    static std::atomic<size_t> opted_dev[kMaxDevices];       /* per instantiation and device: the largest size opted into so far */
    int dev = 0;
    CUDA_TRY(cudaGetDevice(&dev));                           /* the attribute belongs to the current device's context */
    std::atomic<size_t> &opted = opted_dev[dev % kMaxDevices];
    if (opted.load(std::memory_order_relaxed) < smem) {
        CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        opted.store(smem, std::memory_order_relaxed);
    }
    kern<<<grid, kFThreads, smem, s>>>(p);
    CUDA_TRY(cudaGetLastError());
    g_launches.fetch_add(1);
    return ACB_OK;
}

static int launch_pair(const ScanParams &p, int grid, cudaStream_t s) {
    const size_t smem = pair_smem(p.log1, p.log2b).total;
    static std::atomic<size_t> opted_dev[kMaxDevices];
    int dev = 0;
    CUDA_TRY(cudaGetDevice(&dev));
    std::atomic<size_t> &opted = opted_dev[dev % kMaxDevices];
    if (opted.load(std::memory_order_relaxed) < smem) {
        CUDA_TRY(cudaFuncSetAttribute(acb_pair_kernel<17>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        CUDA_TRY(cudaFuncSetAttribute(acb_pair_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        opted.store(smem, std::memory_order_relaxed);
    }
    if (p.log2b == 17) acb_pair_kernel<17><<<grid, kPairThreads, smem, s>>>(p);      /* the 2^20-bit level 1 of 10 k keys and more */
    else acb_pair_kernel<0><<<grid, kPairThreads, smem, s>>>(p);
    CUDA_TRY(cudaGetLastError());
    g_launches.fetch_add(1);
    return ACB_OK;
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
        p.n_tiles = (unsigned int)((p.seg_end - p.seg_begin + kTileBytes - 1) / kTileBytes);
        const int grid = (int)std::min<long long>(tb->sm_count, p.n_tiles);
        int rc = launch_stream(p, tb->filter_flags, tb->stride, grid, s);
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

extern "C" int acb_scan_device(acb_table *tb, const uint8_t *d_hay, int64_t total_bytes,
                               const int64_t *d_offsets, int64_t n_hay, int64_t stride_bytes,
                               acb_match *d_out, int64_t cap, int64_t *d_count, void *stream, int algo) {
    if (!tb || !d_count || total_bytes < 0 || n_hay < 0 || cap < 0 || (cap > 0 && !d_out)) { acb_set_error("bad argument"); return ACB_EINVAL; }
    if (n_hay > 0x7fffffffLL) { acb_set_error("more than 2^31-1 haystacks in one batch"); return ACB_ERANGE; }
    if (!d_offsets) {
        if (stride_bytes <= 0 || stride_bytes % tb->L || stride_bytes * n_hay != total_bytes) {
            acb_set_error("fixed-stride batch needs stride_bytes > 0, a multiple of letter_bytes, and n_hay*stride == total_bytes");
            return ACB_EINVAL;
        }
        if (stride_bytes / tb->L > 0x7fffffffLL) { acb_set_error("haystack longer than 2^31-1 letters"); return ACB_ERANGE; }
    }
    if (total_bytes == 0 || n_hay == 0) return ACB_OK;
    if (reinterpret_cast<uintptr_t>(d_hay) & 15) { acb_set_error("d_hay must be 16-byte aligned"); return ACB_EINVAL; }
    CUDA_TRY(cudaSetDevice(tb->device));
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);

    ScanParams p;
    fill_params(tb, p, d_hay, total_bytes, d_offsets, n_hay, stride_bytes, d_out, cap, d_count);

    if (algo == ACB_ALGO_AUTO) algo = ACB_ALGO_FILTER;
    if (tb->n_keys == 0) return ACB_OK;                     /* empty key set: nothing can match */
    const bool timing = g_timing.load() != 0;
    if (timing) {
        if (!tb->ev0) { CUDA_TRY(cudaEventCreate(&tb->ev0)); CUDA_TRY(cudaEventCreate(&tb->ev1)); }
        CUDA_TRY(cudaEventRecord(tb->ev0, s));
    }
    if (algo == ACB_ALGO_FILTER) {
        int rc = launch_filter_range(tb, p, 0, total_bytes, s);
        if (rc != ACB_OK) return rc;
    } else if (algo == ACB_ALGO_DFA) {
        long long spans = (total_bytes + kDfaSpan - 1) / kDfaSpan;
        long long grid = (spans + kDfaThreads - 1) / kDfaThreads;
        if (grid > 0x7fffffffLL) { acb_set_error("batch too large for one launch"); return ACB_ERANGE; }
        acb_dfa_kernel<<<(unsigned)grid, kDfaThreads, 0, s>>>(p);
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) { acb_set_error("DFA kernel launch failed: %s", cudaGetErrorString(e)); return ACB_ECUDA; }
        g_launches.fetch_add(1);
    } else if (algo == ACB_ALGO_LONG) {
        if (!tb->d_long_final) CUDA_TRY(cudaMalloc(reinterpret_cast<void **>(&tb->d_long_final), sizeof(int32_t)));
        p.long_init = tb->long_init;
        p.long_final = tb->d_long_final;
        tb->long_init = 0;                                      /* one shot */
        long long grid = (n_hay + kDfaThreads - 1) / kDfaThreads;
        acb_long_kernel<<<(unsigned)grid, kDfaThreads, 0, s>>>(p);
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) { acb_set_error("iter_long kernel launch failed: %s", cudaGetErrorString(e)); return ACB_ECUDA; }
        g_launches.fetch_add(1);
    } else {
        acb_set_error("unknown algo %d", algo);
        return ACB_EINVAL;
    }
    if (timing) {
        CUDA_TRY(cudaEventRecord(tb->ev1, s));
        CUDA_TRY(cudaEventSynchronize(tb->ev1));
        float ms = 0.f;
        CUDA_TRY(cudaEventElapsedTime(&ms, tb->ev0, tb->ev1));
        g_last_ms = ms;
    }
    return ACB_OK;
}

extern "C" int acb_table_set_long_state(acb_table *tb, int32_t state) {
    if (!tb || state < 0 || state >= tb->S) { acb_set_error("not a state of this automaton"); return ACB_EINVAL; }
    tb->long_init = state;
    return ACB_OK;
}

extern "C" int acb_table_get_long_state(acb_table *tb, int32_t *state) {
    if (!tb || !state) { acb_set_error("bad argument"); return ACB_EINVAL; }
    *state = 0;
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

/* ------------------------------------------------------------ record sort */
/* Reference order (SURVEY 3.3): haystack, then end_index ascending, then longest key first.  One
 * 64-bit radix key per record: hay_id | end_index | (max_len - len), packed into the fewest bits. */
namespace {
__global__ void acb_sortkey_kernel(const acb_match *rec, long long n, const int32_t *key_len, int be, int bl,
                                   int max_len, unsigned long long *keys) {
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const acb_match m = rec[i];
    const unsigned long long inv = (unsigned long long)(max_len - __ldg(key_len + m.key_id));
    keys[i] = ((unsigned long long)(uint32_t)m.hay_id << (be + bl)) | ((unsigned long long)(uint32_t)m.end_index << bl) | inv;
}
int bits_for(unsigned long long v) { int b = 1; while (b < 64 && (v >> b)) b++; return b; }
} // namespace

extern "C" int acb_sort_matches_device(acb_table *tb, acb_match *d_records, int64_t n, int64_t n_hay,
                                       int64_t max_hay_letters, void *stream) {
    if (!tb || n < 0 || (n && !d_records)) { acb_set_error("bad argument"); return ACB_EINVAL; }
    if (n <= 1) return ACB_OK;
    CUDA_TRY(cudaSetDevice(tb->device));
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    const int max_len = tb->max_key_bytes / tb->L;
    const int bh = bits_for((unsigned long long)std::max<int64_t>(n_hay - 1, 1));
    const int be = bits_for((unsigned long long)std::max<int64_t>(max_hay_letters, 1));
    const int bl = bits_for((unsigned long long)max_len);
    if (bh + be + bl > 64) { acb_set_error("sort key does not fit 64 bits (%d+%d+%d)", bh, be, bl); return ACB_ERANGE; }
    size_t temp = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, temp, (const unsigned long long *)nullptr, (unsigned long long *)nullptr,
                                    (const acb_match *)nullptr, (acb_match *)nullptr, (int)n, 0, bh + be + bl, s);
    const size_t need = (size_t)n * (2 * sizeof(unsigned long long) + sizeof(acb_match)) + temp + 1024;
    if (tb->sort_cap < need) {
        if (tb->d_sort) { cudaFree(tb->d_sort); tb->d_sort = nullptr; tb->sort_cap = 0; }
        CUDA_TRY(cudaMalloc(&tb->d_sort, need + need / 4));
        tb->sort_cap = need + need / 4;
    }
    if (n > 0x7fffffffLL) { acb_set_error("too many records to sort on the device"); return ACB_ERANGE; }
    char *base = reinterpret_cast<char *>(tb->d_sort);
    unsigned long long *k0 = reinterpret_cast<unsigned long long *>(base);
    unsigned long long *k1 = k0 + n;
    acb_match *r1 = reinterpret_cast<acb_match *>(k1 + n);
    void *tmp = reinterpret_cast<void *>((reinterpret_cast<uintptr_t>(r1 + n) + 255) & ~(uintptr_t)255);
    acb_sortkey_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(d_records, n, tb->d_keylen, be, bl, max_len, k0);
    CUDA_TRY(cudaGetLastError());
    g_launches.fetch_add(1);
    CUDA_TRY(cub::DeviceRadixSort::SortPairs(tmp, temp, k0, k1, d_records, r1, (int)n, 0, bh + be + bl, s));
    CUDA_TRY(cudaMemcpyAsync(d_records, r1, (size_t)n * sizeof(acb_match), cudaMemcpyDeviceToDevice, s));
    return ACB_OK;
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
    if (sort) {                                                 /* scratch of the per-chunk sorts, once, before anything is in flight */
        size_t temp = 0;
        cub::DeviceRadixSort::SortPairs(nullptr, temp, (const unsigned long long *)nullptr, (unsigned long long *)nullptr,
                                        (const acb_match *)nullptr, (acb_match *)nullptr, (int)std::min<int64_t>(cap, 0x7fffffff), 0, 64, tb->s_sort);
        const size_t need = (size_t)cap * (2 * sizeof(unsigned long long) + sizeof(acb_match)) + temp + 1024;
        if (tb->sort_cap < need) {
            if (tb->d_sort) { cudaFree(tb->d_sort); tb->d_sort = nullptr; tb->sort_cap = 0; }
            CUDA_TRY(cudaMalloc(&tb->d_sort, need));
            tb->sort_cap = need;
        }
    }
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
        const int32_t *kl = tb->key_len.data();
        auto less = [kl](const acb_match &a, const acb_match &b) {
            if (a.hay_id != b.hay_id) return a.hay_id < b.hay_id;
            if (a.end_index != b.end_index) return a.end_index < b.end_index;
            return kl[a.key_id] > kl[b.key_id];
        };
        for (int c = 0; c + 1 < nch; c++) {
            const unsigned long long mid = tb->h_counts[c];
            if (mid == 0 || mid >= n) continue;
            const int32_t h = tb->h_out[mid - 1].hay_id;          /* the last haystack of chunk c; the cut lies in it or right after it */
            if (tb->h_out[mid].hay_id != h) continue;
            unsigned long long lo = mid, hi = mid;
            while (lo > 0 && tb->h_out[lo - 1].hay_id == h) lo--;
            const unsigned long long stop = std::min<unsigned long long>(n, tb->h_counts[c + 1]);   /* this cut's run ends with chunk c+1; a longer haystack meets the next cut */
            while (hi < stop && tb->h_out[hi].hay_id == h) hi++;
            std::inplace_merge(tb->h_out + lo, tb->h_out + mid, tb->h_out + hi, less);
        }
    }
    tb->h_out_n = n;
    return ACB_OK;
}

extern "C" int acb_scan_host(acb_table *tb, const uint8_t *hay, int64_t total_bytes,
                             const int64_t *offsets, int64_t n_hay, int64_t stride_bytes,
                             acb_match *out, int64_t cap, int64_t *n_found, int algo, int sort) {
    if (!tb || !n_found || total_bytes < 0 || n_hay < 0 || cap < 0) { acb_set_error("bad argument"); return ACB_EINVAL; }
    *n_found = 0;
    tb->h_out_n = 0;
    if (total_bytes == 0 || n_hay == 0) return ACB_OK;
    CUDA_TRY(cudaSetDevice(tb->device));
    if (!tb->stream) CUDA_TRY(cudaStreamCreateWithFlags(&tb->stream, cudaStreamNonBlocking));
    if (!tb->w_count) CUDA_TRY(cudaMalloc(reinterpret_cast<void **>(&tb->w_count), sizeof(unsigned long long)));
    if (!tb->h_count) CUDA_TRY(cudaMallocHost(reinterpret_cast<void **>(&tb->h_count), sizeof(unsigned long long)));
    int rc;
    if ((rc = ensure(&tb->w_hay, &tb->w_hay_cap, (size_t)total_bytes + 64))) return rc;
    if (offsets && (rc = ensure(&tb->w_off, &tb->w_off_cap, (size_t)n_hay + 1))) return rc;
    if ((rc = ensure(&tb->w_out, &tb->w_out_cap, (size_t)std::max<int64_t>(cap, 1)))) return rc;
    cudaStream_t s = tb->stream;
    {   /* large batches on the fast path: copy, scan, sort and copy-back as a pipeline over chunks */
        const int64_t max_letters = (offsets ? total_bytes : stride_bytes) / tb->L;
        const int bits = bits_for((unsigned long long)std::max<int64_t>(n_hay - 1, 1)) + bits_for((unsigned long long)std::max<int64_t>(max_letters, 1)) +
                         bits_for((unsigned long long)(tb->max_key_bytes / tb->L));
        static const bool no_pipe = getenv("ACB_NO_PIPELINE") != nullptr;
        if (!no_pipe && (algo == ACB_ALGO_AUTO || algo == ACB_ALGO_FILTER) && tb->n_keys > 0 && total_bytes >= (48LL << 20) && bits <= 64 && cap < 0x7fffffffLL) {
            rc = scan_host_pipelined(tb, hay, total_bytes, offsets, n_hay, stride_bytes, cap, n_found, sort);
            if (rc == ACB_OK && out && *n_found) memcpy(out, tb->h_out, (size_t)*n_found * sizeof(acb_match));
            return rc;
        }
    }
    static const bool trace = getenv("ACB_TRACE") != nullptr;          /* phase timing to stderr (adds syncs) */
    auto now = [] { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
    double t0 = trace ? now() : 0, t1 = 0, t2 = 0, t3 = 0, t4 = 0;
    CUDA_TRY(cudaMemcpyAsync(tb->w_hay, hay, (size_t)total_bytes, cudaMemcpyHostToDevice, s));
    if (offsets) CUDA_TRY(cudaMemcpyAsync(tb->w_off, offsets, (size_t)(n_hay + 1) * sizeof(long long), cudaMemcpyHostToDevice, s));
    CUDA_TRY(cudaMemsetAsync(tb->w_count, 0, sizeof(unsigned long long), s));
    if (trace) { cudaStreamSynchronize(s); t1 = now(); }
    rc = acb_scan_device(tb, tb->w_hay, total_bytes, offsets ? reinterpret_cast<const int64_t *>(tb->w_off) : nullptr,
                         n_hay, stride_bytes, tb->w_out, cap, reinterpret_cast<int64_t *>(tb->w_count), s, algo);
    if (rc != ACB_OK) return rc;
    CUDA_TRY(cudaMemcpyAsync(tb->h_count, tb->w_count, sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    if (trace) t2 = now();
    unsigned long long n = *tb->h_count;
    *n_found = (int64_t)n;
    if (n > (unsigned long long)cap) {
        acb_set_error("match buffer too small: %llu matches, capacity %lld", n, (long long)cap);
        return ACB_EOVERFLOW;
    }
    if (n) {
        if (tb->h_out_cap < n) {                               /* pinned staging: D2H at full PCIe rate */
            if (tb->h_out) { acb_release_records(tb->h_out, (int64_t)tb->h_out_cap); tb->h_out = nullptr; tb->h_out_cap = 0; }
            size_t got = 0;
            if (acb_match *p = pool_take((size_t)n, &got)) {  /* a buffer some caller has given back */
                tb->h_out = p;
                tb->h_out_cap = got;
            } else {
                size_t want = (size_t)n + (size_t)n / 4 + 1024;
                CUDA_TRY(cudaMallocHost(reinterpret_cast<void **>(&tb->h_out), want * sizeof(acb_match)));
                tb->h_out_cap = want;
            }
        }
        bool host_sort = sort != 0;
        if (sort) {                                            /* radix sort on the device when the key fits 64 bits */
            const int64_t max_letters = (offsets ? total_bytes : stride_bytes) / tb->L;
            if (acb_sort_matches_device(tb, tb->w_out, (int64_t)n, n_hay, max_letters, s) == ACB_OK) host_sort = false;
        }
        if (trace) { cudaStreamSynchronize(s); t3 = now(); }
        CUDA_TRY(cudaMemcpyAsync(tb->h_out, tb->w_out, (size_t)n * sizeof(acb_match), cudaMemcpyDeviceToHost, s));
        CUDA_TRY(cudaStreamSynchronize(s));
        if (host_sort) {
            const int32_t *kl = tb->key_len.data();
            std::sort(tb->h_out, tb->h_out + n, [kl](const acb_match &a, const acb_match &b) {
                if (a.hay_id != b.hay_id) return a.hay_id < b.hay_id;
                if (a.end_index != b.end_index) return a.end_index < b.end_index;
                return kl[a.key_id] > kl[b.key_id];            /* longest first: fail-chain order */
            });
        }
        if (out) memcpy(out, tb->h_out, (size_t)n * sizeof(acb_match));   /* out == NULL: fetch with acb_copy_records */
    }
    tb->h_out_n = n;
    if (trace) {
        t4 = now();
        fprintf(stderr, "[acb_scan_host] %lld B: h2d %.3f ms, scan %.3f ms, sort %.3f ms, d2h+copy %.3f ms (%llu records)\n",
                (long long)total_bytes, t1 - t0, t2 - t1, t3 ? t3 - t2 : 0.0, t3 ? t4 - t3 : t4 - t2, n);
    }
    return ACB_OK;
}

