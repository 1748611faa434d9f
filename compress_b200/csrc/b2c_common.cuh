// compress_b200/csrc/b2c_common.cuh -- device-side utilities shared by all kernels:
// warp/block scans, named barriers, unaligned shared-memory loads, the
// cooperative bit-run writer, 1-D TMA bulk loads.  sm_90a (Hopper) and later.
//
// The same sources also compile under tests/emu/simt_emu.h (B2C_EMU) so kernel
// logic can be exercised on the GPU-less dev box; that build is test
// infrastructure and is never part of libb200comp.so.
#pragma once
#ifdef B2C_EMU
#include "simt_emu.h"
#else
#include <cuda_runtime.h>
#include <cstdint>
#endif

#define B2C_DEV __device__ __forceinline__
// read-only global load (data written by an earlier kernel): lets the compiler batch loads across loop iterations
#ifdef B2C_EMU
#define B2C_LDG(p) (*(p))
#else
#define B2C_LDG(p) __ldg(p)
#endif
#define FULLMASK 0xffffffffu

namespace b2c {

B2C_DEV unsigned lane_id() { return threadIdx.x & 31; }
B2C_DEV unsigned warp_id() { return threadIdx.x >> 5; }
B2C_DEV uint32_t highbit32(uint32_t v) { return 31u - (uint32_t)__clz((int)v); }  // v != 0
// Profiling stamp: lane 0 stores clock64 at row[k] (nothing without a row, and nothing in the emulator build).
B2C_DEV void stamp_clock(unsigned long long *row, int k) {
#ifndef B2C_EMU
    if (row && lane_id() == 0) row[k] = (unsigned long long)clock64();
#endif
}

// Named barrier over a warp-multiple subset of the CTA (id 1..15; 0 is __syncthreads).
B2C_DEV void bar_sync(int id, int nthreads) {
#ifdef B2C_EMU
    emu_named_barrier(id, nthreads);
#else
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
#endif
}

// Barrier over a thread group: bar_id 0 = whole CTA, 1..15 = named barrier over nthreads, < 0 = one warp.
B2C_DEV void group_sync(int bar_id, int nthreads) {
    if (bar_id == 0) __syncthreads();
    else if (bar_id < 0) __syncwarp();
    else bar_sync(bar_id, nthreads);
}

// ---- unaligned little-endian loads from a 4-byte aligned base (shared or global).
// Reads the aligned words covering [pos, pos+len); the buffer must be padded.
B2C_DEV uint32_t ld32u(const uint8_t *base, uint32_t pos) {
    const uint32_t *w = reinterpret_cast<const uint32_t *>(base + (pos & ~3u));
    uint32_t sh = (pos & 3u) * 8u;
    uint32_t a = w[0];
    if (sh == 0) return a;
    return __funnelshift_r(a, w[1], sh);
}
B2C_DEV uint64_t ld64u(const uint8_t *base, uint32_t pos) {
    const uint32_t *w = reinterpret_cast<const uint32_t *>(base + (pos & ~3u));
    uint32_t sh = (pos & 3u) * 8u;
    uint32_t a = w[0], b = w[1];
    if (sh == 0) return ((uint64_t)b << 32) | a;
    uint32_t c = w[2];
    return ((uint64_t)__funnelshift_r(b, c, sh) << 32) | __funnelshift_r(a, b, sh);
}

// ---- warp scans (inclusive) ----
B2C_DEV uint32_t warp_scan_incl(uint32_t v) {
    unsigned lane = lane_id();
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        uint32_t t = __shfl_up_sync(FULLMASK, v, d);
        if (lane >= (unsigned)d) v += t;
    }
    return v;
}
B2C_DEV uint32_t warp_sum(uint32_t v) {
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(FULLMASK, v, d);
    return v;
}
B2C_DEV uint32_t warp_max(uint32_t v) {
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
        uint32_t t = __shfl_xor_sync(FULLMASK, v, d);
        v = t > v ? t : v;
    }
    return v;
}

// Exclusive scan of one value per thread across `nthreads` (multiple of 32, <= 1024) threads
// that all call this with the same barrier id.  ws: shared scratch of >= 33 uint32.
// Returns the exclusive prefix; *total receives the sum over all threads.
B2C_DEV uint32_t group_scan_excl(uint32_t v, uint32_t *ws, int bar_id, int nthreads, unsigned tid_in_group,
                                 uint32_t *total) {
    unsigned lane = tid_in_group & 31, w = tid_in_group >> 5;
    uint32_t incl = warp_scan_incl(v);
    if (lane == 31) ws[w] = incl;
    group_sync(bar_id, nthreads);
    if (w == 0) {
        int nw = nthreads >> 5;
        uint32_t x = (lane < (unsigned)nw) ? ws[lane] : 0;
        uint32_t xi = warp_scan_incl(x);
        ws[lane] = xi - x;  // exclusive warp bases
        if (lane == 31) ws[32] = xi;
    }
    group_sync(bar_id, nthreads);
    uint32_t base = ws[w];
    *total = ws[32];
    // callers must place a barrier before reusing ws
    return base + incl - v;
}

B2C_DEV uint32_t warp_scan_incl_max(uint32_t v) {
    unsigned lane = lane_id();
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        uint32_t t = __shfl_up_sync(FULLMASK, v, d);
        if (lane >= (unsigned)d && t > v) v = t;
    }
    return v;
}
// Exclusive prefix maximum (identity 0) with the same calling convention as group_scan_excl; *total = overall maximum.
B2C_DEV uint32_t group_scan_excl_max(uint32_t v, uint32_t *ws, int bar_id, int nthreads, unsigned tid_in_group,
                                     uint32_t *total) {
    unsigned lane = tid_in_group & 31, w = tid_in_group >> 5;
    uint32_t incl = warp_scan_incl_max(v);
    uint32_t excl = __shfl_up_sync(FULLMASK, incl, 1);
    if (lane == 0) excl = 0;
    group_sync(bar_id, nthreads);      // ws may still be read by a previous scan
    if (lane == 31) ws[w] = incl;
    group_sync(bar_id, nthreads);
    if (w == 0) {
        int nw = nthreads >> 5;
        uint32_t x = (lane < (unsigned)nw) ? ws[lane] : 0;
        uint32_t xi = warp_scan_incl_max(x);
        uint32_t xe = __shfl_up_sync(FULLMASK, xi, 1);
        if (lane == 0) xe = 0;
        ws[lane] = xe;  // exclusive warp bases
        if (lane == 31) ws[32] = xi;
    }
    group_sync(bar_id, nthreads);
    uint32_t base = ws[w];
    *total = ws[32];
    return base > excl ? base : excl;
}

// ---- cooperative bit-run writer ----
// Many threads append disjoint, contiguous bit ranges of one little-endian,
// LSB-first bitstream held in zero-initialised shared memory (32-bit words).
// Words wholly inside a thread's range are stored plainly; the first and last
// (possibly shared) words are merged with atomicOr.
struct BitRun {
    uint32_t *words;   // stream base (4-byte aligned)
    uint32_t bitpos;   // absolute bit position of the next bit to add
    uint64_t acc;      // pending bits, LSB = bit `wordbit` of the current word
    uint32_t nacc;     // number of pending bits in acc (including the leading offset)
    uint32_t widx;     // index of the current (unflushed) word
    bool first;        // the current word is the first word of this run

    B2C_DEV void init(uint32_t *w, uint32_t startbit) {
        words = w; bitpos = startbit; widx = startbit >> 5; nacc = startbit & 31; acc = 0; first = true;
    }
    B2C_DEV void flush_word() {
        uint32_t wv = (uint32_t)acc;
        if (first) { if (wv) atomicOr(&words[widx], wv); first = false; }
        else words[widx] = wv;
        widx++; acc >>= 32; nacc -= 32;
    }
    // add up to 32 bits (value must already be masked to nbits)
    B2C_DEV void add(uint32_t value, uint32_t nbits) {
        acc |= (uint64_t)value << nacc;
        nacc += nbits; bitpos += nbits;
        if (nacc >= 32) flush_word();
    }
    B2C_DEV void finish() {
        if (nacc > 0) {
            uint32_t wv = (uint32_t)acc;
            if (wv) atomicOr(&words[widx], wv);
        }
    }
};

// XXH64: merge of the four accumulators, the tail bytes and the avalanche (xxhash.go:101-160)
B2C_DEV uint64_t xxh64_finish(uint64_t v1, uint64_t v2, uint64_t v3, uint64_t v4, const uint8_t *src, uint64_t n) {
    const uint64_t P1 = 11400714785074694791ull, P2 = 14029467366897019727ull, P3 = 1609587929392839161ull,
                   P4 = 9650029242287828579ull, P5 = 2870177450012600261ull;
    uint64_t h;
    uint64_t p = (n / 32) * 32;
    if (n >= 32) {
        h = ((v1 << 1) | (v1 >> 63)) + ((v2 << 7) | (v2 >> 57)) + ((v3 << 12) | (v3 >> 52)) + ((v4 << 18) | (v4 >> 46));
#define XMERGE(vv)                                                                                     \
    do {                                                                                               \
        uint64_t t_ = (vv) * P2; t_ = (t_ << 31) | (t_ >> 33); t_ *= P1;                               \
        h ^= t_; h = h * P1 + P4;                                                                      \
    } while (0)
        XMERGE(v1); XMERGE(v2); XMERGE(v3); XMERGE(v4);
#undef XMERGE
    } else {
        h = P5;
    }
    h += n;
    while (p + 8 <= n) {
        uint64_t k1 = 0;
        for (int b = 0; b < 8; b++) k1 |= (uint64_t)src[p + b] << (8 * b);
        k1 *= P2; k1 = (k1 << 31) | (k1 >> 33); k1 *= P1;
        h ^= k1; h = ((h << 27) | (h >> 37)) * P1 + P4;
        p += 8;
    }
    if (p + 4 <= n) {
        uint32_t k4 = 0;
        for (int b = 0; b < 4; b++) k4 |= (uint32_t)src[p + b] << (8 * b);
        h ^= (uint64_t)k4 * P1;
        h = ((h << 23) | (h >> 41)) * P2 + P3;
        p += 4;
    }
    while (p < n) {
        h ^= (uint64_t)src[p] * P5;
        h = ((h << 11) | (h >> 53)) * P1;
        p++;
    }
    h ^= h >> 33; h *= P2; h ^= h >> 29; h *= P3; h ^= h >> 32;
    return h;
}

// XXH64 (zstd/internal/xxhash/xxhash.go:62-160) of src[0, n): four adjacent lanes (q = 0..3, the first of them lane
// quadBaseLane of the warp) hold the four accumulators; all four must call (with n = 0 when they have no input); the
// digest is returned on q == 0.
B2C_DEV uint64_t xxh64_quad(const uint8_t *src, uint64_t n, unsigned q /*0..3*/, unsigned quadBaseLane) {
    const uint64_t P1 = 11400714785074694791ull, P2 = 14029467366897019727ull, P3 = 1609587929392839161ull,
                   P4 = 9650029242287828579ull, P5 = 2870177450012600261ull;
    const bool aligned = (reinterpret_cast<uintptr_t>(src) & 7) == 0;
    uint64_t v = (q == 0) ? P1 + P2 : (q == 1) ? P2 : (q == 2) ? 0ull : (0ull - P1);
    const uint64_t stripes = n / 32;
    uint64_t i = 0;
    if (aligned) {
        // sixteen stripes per batch: the loads are independent of the accumulator, so they are all in flight while
        // the (serial) multiply-rotate chain of the previous ones runs
        const uint64_t *s8 = reinterpret_cast<const uint64_t *>(src) + q;
        for (; i + 16 <= stripes; i += 16) {
            uint64_t in[16];
#pragma unroll
            for (int k = 0; k < 16; k++) in[k] = s8[4 * (i + k)];
#pragma unroll
            for (int k = 0; k < 16; k++) {
                v += in[k] * P2;
                v = (v << 31) | (v >> 33);
                v *= P1;
            }
        }
    }
    for (; i < stripes; i++) {
        uint64_t in;
        if (aligned) in = reinterpret_cast<const uint64_t *>(src)[4 * i + q];
        else { in = 0; for (int b = 0; b < 8; b++) in |= (uint64_t)src[32 * i + 8 * q + b] << (8 * b); }
        v += in * P2;
        v = (v << 31) | (v >> 33);
        v *= P1;
    }
    uint64_t v1 = __shfl_sync(FULLMASK, v, quadBaseLane), v2 = __shfl_sync(FULLMASK, v, quadBaseLane + 1),
             v3 = __shfl_sync(FULLMASK, v, quadBaseLane + 2), v4 = __shfl_sync(FULLMASK, v, quadBaseLane + 3);
    if (q != 0) return 0;
    return xxh64_finish(v1, v2, v3, v4, src, n);
}

// XXH64 of a long input by ONE WARP: all lanes stream the input (coalesced 16-byte loads, the next 2 KiB tile requested
// while the current one is hashed) into a warp-private shared buffer, lanes 0-3 run the four accumulator chains over it.
// The digest is a serial recurrence, so a lane-quad on its own waits out one memory round trip per handful of stripes;
// here the loads of the whole warp are in flight instead.  stg: 2 x 2 KiB per warp, 16-byte aligned.  src 16-byte
// aligned (else the quad form is used).  Result on lane 0.
constexpr uint32_t XXH_TILE = 2048;
B2C_DEV uint64_t xxh64_warp(const uint8_t *src, uint64_t n, uint8_t *stg, unsigned lane) {
    const uint64_t P1 = 11400714785074694791ull, P2 = 14029467366897019727ull;
    if ((reinterpret_cast<uintptr_t>(src) & 15) != 0) return xxh64_quad(src, lane < 4 ? n : 0, lane & 3, lane & ~3u);
    uint64_t v = (lane == 0) ? P1 + P2 : (lane == 1) ? P2 : (lane == 2) ? 0ull : (0ull - P1);
    const uint64_t ntiles = n / XXH_TILE;
    const uint4 *g = reinterpret_cast<const uint4 *>(src);
    uint4 r[4];
    if (ntiles) {
#pragma unroll
        for (int k = 0; k < 4; k++) r[k] = B2C_LDG(g + k * 32 + lane);
    }
    for (uint64_t t = 0; t < ntiles; t++) {
        uint4 *sb = reinterpret_cast<uint4 *>(stg + (t & 1) * XXH_TILE);
#pragma unroll
        for (int k = 0; k < 4; k++) sb[k * 32 + lane] = r[k];
        if (t + 1 < ntiles) {
#pragma unroll
            for (int k = 0; k < 4; k++) r[k] = B2C_LDG(g + (t + 1) * (XXH_TILE / 16) + k * 32 + lane);
        }
        __syncwarp();
        if (lane < 4) {
            const uint64_t *s8 = reinterpret_cast<const uint64_t *>(sb) + lane;
#pragma unroll 8
            for (uint32_t i = 0; i < XXH_TILE / 32; i++) {
                v += s8[4 * i] * P2;
                v = (v << 31) | (v >> 33);
                v *= P1;
            }
        }
        __syncwarp();      // (the buffer written two tiles later is this one)
    }
    // the stripes behind the last whole tile: straight from memory
    const uint64_t done = ntiles * XXH_TILE, stripes = n / 32;
    if (lane < 4)
        for (uint64_t i = done / 32; i < stripes; i++) {
            v += reinterpret_cast<const uint64_t *>(src)[4 * i + lane] * P2;
            v = (v << 31) | (v >> 33);
            v *= P1;
        }
    const uint64_t v1 = __shfl_sync(FULLMASK, v, 0), v2 = __shfl_sync(FULLMASK, v, 1), v3 = __shfl_sync(FULLMASK, v, 2),
                   v4 = __shfl_sync(FULLMASK, v, 3);
    if (lane != 0) return 0;
    return xxh64_finish(v1, v2, v3, v4, src, n);
}

// Cooperative copy of sz bytes between arbitrarily aligned global addresses: bytes up to the destination's 16-byte boundary,
// then 4-byte destination words assembled from aligned source words, then the tail.  All threads of the group call.
B2C_DEV void coop_copy(uint8_t *d, const uint8_t *s, uint32_t sz, unsigned tid, unsigned nthreads) {
    uint32_t head = (uint32_t)((16 - (reinterpret_cast<uintptr_t>(d) & 15)) & 15);
    if (head > sz) head = sz;
    for (uint32_t i = tid; i < head; i += nthreads) d[i] = s[i];
    const uint32_t body = (sz - head) & ~3u;
    for (uint32_t i = tid * 4; i < body; i += nthreads * 4) *reinterpret_cast<uint32_t *>(d + head + i) = ld32u(s, head + i);
    for (uint32_t i = head + body + tid; i < sz; i += nthreads) d[i] = s[i];
}

// Execute up to 32 matches (lane i: copy myML bytes from out + myDst - myMO to out + myDst; mine = this lane has one), whose
// destinations increase with the lane: in waves -- a match runs once its source ends before the destination of every pending
// match; short ones as per-lane word copies, long ones (>= 64 bytes) by the whole warp.  All lanes call.
B2C_DEV void lz_exec_match_waves(uint8_t *out, bool mine, uint32_t myDst, uint32_t myMO, uint32_t myML, unsigned lane) {
    // ---- matches in waves: a match runs once its source ends before the destination of every pending match
    bool pending = mine;
    const uint32_t srcEnd = (myMO >= myML) ? myDst - myMO + myML : myDst;   // self-overlap: source ends at dst
    for (;;) {
        const uint32_t minDst = __reduce_min_sync(FULLMASK, pending ? myDst : 0xffffffffu);
        if (minDst == 0xffffffffu) break;
        const bool ready = pending && (srcEnd <= minDst || myDst == minDst);
        const bool longM = ready && myML >= 64;
        if (ready && !longM) {
            const uint8_t *from = out + myDst - myMO;
            uint8_t *to = out + myDst;
            if (myMO >= 8 || myMO >= myML) {
                // Word copy: bytes up to the destination's 4-byte boundary, then aligned destination words whose
                // source words are assembled from aligned loads with a funnel shift (one new load per word), then
                // the last bytes.  A source word is read at most 7 bytes ahead of the byte being produced, so with a
                // distance of 8 or more (or no overlap at all) everything it holds that is used is final.
                uint32_t k = (uint32_t)((4 - (reinterpret_cast<uintptr_t>(to) & 3)) & 3);
                if (k > myML) k = myML;
                for (uint32_t q = 0; q < k; q++) to[q] = from[q];
                const uint32_t nw = (myML - k) >> 2;
                if (nw) {
                    const uint8_t *f = from + k;
                    const uint32_t fa = (uint32_t)(reinterpret_cast<uintptr_t>(f) & 3), sh = fa * 8;
                    const uint32_t *fw = reinterpret_cast<const uint32_t *>(f - fa);
                    uint32_t *tw = reinterpret_cast<uint32_t *>(to + k);
                    if (sh == 0) {
                        for (uint32_t i = 0; i < nw; i++) tw[i] = fw[i];
                    } else {
                        uint32_t w0 = fw[0];
                        for (uint32_t i = 0; i < nw; i++) {
                            const uint32_t w1 = fw[i + 1];
                            tw[i] = __funnelshift_r(w0, w1, sh);
                            w0 = w1;
                        }
                    }
                    k += nw * 4;
                }
                for (; k < myML; k++) to[k] = from[k];
            } else {
                for (uint32_t k = 0; k < myML; k++) to[k] = from[k];
            }
        }
        for (unsigned m = __ballot_sync(FULLMASK, longM); m; m &= m - 1) {
            const int f = __ffs((int)m) - 1;
            const uint32_t fd = __shfl_sync(FULLMASK, myDst, f);
            const uint32_t fo = __shfl_sync(FULLMASK, myMO, f), fn = __shfl_sync(FULLMASK, myML, f);
            const uint8_t *from = out + fd - fo;
            if (fo >= fn || fo >= 32) {
                for (uint32_t k0 = 0; k0 < fn; k0 += 32) {
                    const uint32_t k = k0 + lane;
                    if (k < fn) out[fd + k] = from[k];
                    if (fo < fn) __syncwarp();
                }
            } else {
                for (uint32_t k = lane; k < fn; k += 32) out[fd + k] = from[k % fo];
            }
            __syncwarp();
        }
        if (ready) pending = false;
        __syncwarp();
    }
}

// streaming (evict-first) 8-byte store: data another kernel reads once should not push reused lines out of L2
B2C_DEV void st_stream64(uint64_t *p, uint64_t v) {
#ifndef B2C_EMU
    __stcs(reinterpret_cast<unsigned long long *>(p), (unsigned long long)v);
#else
    *p = v;
#endif
}
// hint: bring the 128-byte line holding p into L1 (no-op under the emulator)
B2C_DEV void prefetch_l1(const void *p) {
#ifndef B2C_EMU
    asm volatile("prefetch.global.L1 [%0];" ::"l"(p));
#else
    (void)p;
#endif
}

// read-only 32-bit load of data that is re-read all through a kernel while other data streams past it: an L2 cache
// policy (createpolicy ... evict_last) keeps it resident.  pol = l2_keep_policy(), once per thread.
B2C_DEV uint64_t l2_keep_policy() {
#ifndef B2C_EMU
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
    return pol;
#else
    return 0;
#endif
}
B2C_DEV uint32_t ld_keep32(const uint32_t *p, uint64_t pol) {
#ifndef B2C_EMU
    uint32_t v;
    asm volatile("ld.global.nc.L2::cache_hint.u32 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(pol));
    return v;
#else
    (void)pol;
    return *p;
#endif
}
// 32-bit load that is cached in L2 only: with most of the SM's memory configured as shared memory the few L1 lines
// left cannot hold the lines of hundreds of independent streams, and allocating them serialises the misses
B2C_DEV uint32_t ld_cg32(const uint32_t *p) {
#ifndef B2C_EMU
    return __ldcg(p);
#else
    return *p;
#endif
}
// hint: bring the sector holding p into L2
B2C_DEV void prefetch_l2(const void *p) {
#ifndef B2C_EMU
    asm volatile("prefetch.global.L2 [%0];" ::"l"(p));
#else
    (void)p;
#endif
}

#ifndef B2C_EMU
// ---- 1-D TMA bulk copy global -> shared with mbarrier completion (UBLKCP) ----
B2C_DEV uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
B2C_DEV void mbar_init(uint64_t *bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
B2C_DEV void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
B2C_DEV void mbar_expect_tx(uint64_t *bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
B2C_DEV void tma_load_1d(void *dst_smem, const void *src_gmem, unsigned bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
B2C_DEV void mbar_wait(uint64_t *bar, unsigned phase) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t}" ::"r"(smem_u32(bar)),
        "r"(phase)
        : "memory");
}
#endif

}  // namespace b2c
