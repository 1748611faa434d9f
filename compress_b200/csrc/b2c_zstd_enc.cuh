// compress_b200/csrc/b2c_zstd_enc.cuh -- zstd chunk encoder for sm_90a: entropy stages, framing, work records.
//
// Turns N independent chunks (<= 64 KiB at level 1, <= 128 KiB at levels 2-3) into N complete zstd frames (what one zstd.Encoder.EncodeAll call does
// per chunk, zstd/encoder.go:722-839) or bare blocks.  Replaces, for the GPU path, the reference's
//   zstd/enc_fast.go:294-531  fastEncoder.EncodeNoHist      (match finding)
//   zstd/blockenc.go:481-826  blockEnc.encode               (entropy stage, byte-identical here)
//   zstd/frameenc.go:25-92    frameHeader.appendTo
//   zstd/internal/xxhash      XXH64 frame checksum
//
// Design: a pipeline of six kernels on one stream, each shaped after the parallelism its stage really has, with
// a per-chunk work record (ChunkWork header + a slab of the work pool) in HBM/L2 between them:
//   K1 parse    b2c_lz.cuh: the tile-ordered match finder (levels 1-3; also the S2 / Snappy block encoders)
//   hist        b2c_lz.cuh: literal and sequence-code histograms
//   K2 tables   one 4-warp CTA per chunk: the Huffman table (reference tie-breaking) and the three FSE
//               tables are tiny serial problems -- thousands of them run side by side.
//   K3 chains   one LANE per (chunk, tANS chain): the reference's serial state walk, 32 chunks per warp.
//   K4 pack     one CTA per chunk: code-length / bit-count prefix sums, every thread packs its own bit
//               range of the 4 Huffman streams and of the sequence bitstream into a staging buffer,
//               headers, one coalesced write-back (raw / RLE block fallbacks included).
//   K5 xxh64    four lanes per chunk (the four XXH64 accumulators).
// The parse differs from the reference's serial greedy parse; the entropy stage is byte-identical to
// blockEnc.encode for the same (literals, sequences) -- tests/check_util.py verifies both properties.
// This file: work record and pool layout, S2 tag emitters, K2..K5.
#pragma once
#include "b2c_common.cuh"
#include "b2c_fse.cuh"
#include "b2c_huff.cuh"
#include "b2c_seq.cuh"

namespace b2c {

constexpr uint32_t ENC_MAX_CHUNK = 1u << 16;   // block size of zstd level 1 and of the S2 block encoders
#ifndef PACK_THREADS
#define PACK_THREADS 512
#endif
#ifndef PACK_BITS_LUT
#define PACK_BITS_LUT 1      // extra-bit counts from a 2 x 64 byte shared-memory table instead of compare chains
#endif
#ifndef PACK_MIN_CTAS
#define PACK_MIN_CTAS 2   // two CTAs per SM: caps the kernel at 64 registers per thread
#endif
constexpr int PACK_NT = PACK_THREADS;     // K4 threads per CTA (a multiple of 128: four Huffman streams)
static_assert(PACK_NT % 128 == 0 && PACK_NT >= 384, "K4 loads the Huffman table description with one thread per byte");

enum { ENC_FLAG_CRC = 1, ENC_FLAG_FRAME = 2 };

// Per-chunk work record handed from kernel to kernel (global memory, L2 resident for the active chunks): a small
// header (this struct) plus one slab of the work pool holding the arrays whose size depends on the block size
// (literals, per-sequence values, codes, state bits; layout below, sized by the host per level).
struct alignas(16) ChunkWork {
    uint32_t n, nseq, nlit, kind;          // kind: 0 compressed candidate, 1 raw block, 2 RLE block, 3 too big
    uint32_t rleLen, hufStatus, hufTableLog, tableDescLen;
    uint32_t maxSym[3], pad0;
    uint32_t mode[3], pad1;                // 0 predefined, 1 RLE, 2 FSE
    uint32_t ncountLen[3], pad2;
    uint32_t finalState[3], pad3;
    unsigned long long xxh;
    uint32_t litHist[256];
    uint32_t seqHist[3][64];
    uint16_t ctVal[256];
    uint8_t ctBits[256];
    uint8_t tableDesc[320];
    uint8_t ncount[3][96];
    FseCTable tbl[3];                      // the table each chain uses (new, predefined copy, or RLE)
};

// Frame mode (b2c_zstd_encode_frames_*): chunk i is block `i` of the batch's block list -- `len` bytes at src_base + off,
// preceded (in the same frame, contiguous in memory) by `hist` bytes the match finder may refer to (fastBase.hist /
// addBlock, zstd/enc_base.go:57-199).  Bit 0 of flags: last block of its frame (blockHeader.setLast, blockenc.go:120).
struct EncBlockDesc {
    uint64_t off;
    uint32_t len, hist, frame, flags;
};

struct ZstdEncParams {
    const EncBlockDesc *desc;     // frame mode: block descriptors (then src_stride / src_sizes are unused); else nullptr
    const uint8_t *src_base;      // chunk i at src_base + i * src_stride
    uint64_t src_stride;
    const uint32_t *src_sizes;    // per-chunk sizes (<= 65536); nullptr => all chunks are src_size_all
    uint32_t src_size_all;
    uint8_t *dst_base;
    uint64_t dst_stride;
    uint32_t dst_cap;             // capacity of every destination slot
    int64_t *out_sizes;           // bytes written per chunk, negative = error
    uint32_t nchunks;
    uint32_t flags;
    uint8_t *scratch;             // per-CTA parse scratch: gridDim.x(K1) * LzLayout<..>::SCRATCH_BYTES
    ChunkWork *work;              // [nchunks]
    uint8_t *pool;                // [nchunks] slabs of pool_stride bytes: lit | seqOF | seqLL | seqML | codes[3] | stb[3]
    uint64_t pool_stride;
    uint32_t maxseq;              // capacity of the per-sequence arrays (multiple of 16)
    uint32_t blockmax;            // largest block this launch accepts (65536 or 131072)
    uint32_t big;                 // 1: litLen / matchLen arrays are u32 (blocks > 64 KiB), 0: u16
    uint32_t level;               // 1 fastest, 2 default
    uint64_t src_total;           // non-zero: the chunks tile one buffer of src_total bytes (the last chunk is shorter)
    uint32_t *counter;            // persistent parse kernels: next chunk to hand out (zeroed before the launch)
    uint32_t chunk0;              // sub-batch offset: kernels work on chunks [chunk0, chunk0 + nchunks) of the call
    // optional debug dump (tests): per chunk {nseq, nlit, kind, litMode} + seq triples + literals
    uint32_t *dbg_hdr;            // [nchunks][4]
    uint32_t *dbg_seqs;           // [nchunks][dbg_seq_cap][3]
    uint8_t *dbg_lits;            // [nchunks][65536]
    uint32_t dbg_seq_cap;
    unsigned long long *dbg_cycles;  // optional [nchunks][16][32] per-warp stamps inside K1 and K4 (clock64)
};

#ifdef B2C_EMU
#define B2C_PHASE(k) do { } while (0)
#else
// Every warp's lane 0 stamps clock64 right after each barrier.  BAR.SYNC does not block at issue, so the stamp
// captures the warp's ARRIVAL time at the preceding barrier; the release time is the maximum over warps.
#define B2C_PHASE(k)                                                                                   \
    do {                                                                                               \
        if (P.dbg_cycles && (threadIdx.x & 31) == 0)                                                   \
            P.dbg_cycles[((uint64_t)chunk * 16 + (k)) * 32 + (threadIdx.x >> 5)] = (unsigned long long)clock64(); \
    } while (0)
#endif
// The same stamps in K4 (tools/pack_phase_times.py): its warps take columns 16..31 of the chunk's rows, beside the
// parse's 16 warps, so one timed run records both kernels.  Not every stamp follows a barrier here.
#ifdef B2C_EMU
#define B2C_PACK_PHASE(k) do { } while (0)
#else
#define B2C_PACK_PHASE(k)                                                                              \
    do {                                                                                               \
        if (P.dbg_cycles && (threadIdx.x & 31) == 0 && (threadIdx.x >> 5) < 16)                        \
            P.dbg_cycles[((uint64_t)chunk * 16 + (k)) * 32 + 16 + (threadIdx.x >> 5)] = (unsigned long long)clock64(); \
    } while (0)
#endif
// The same stamps in the hist kernel (tools/hist_phase_times.py): warp w takes row 12 + w, columns 8..15 (beside the
// tables kernel's columns 0..7 of those rows).
#ifdef B2C_EMU
#define B2C_HIST_PHASE(k) do { } while (0)
#else
#define B2C_HIST_PHASE(k)                                                                              \
    do {                                                                                               \
        if (P.dbg_cycles && (threadIdx.x & 31) == 0)                                                   \
            P.dbg_cycles[((uint64_t)chunk * 16 + 12 + (threadIdx.x >> 5)) * 32 + 8 + (k)] = (unsigned long long)clock64(); \
    } while (0)
#endif
// The same stamps in K2 (tools/tables_phase_times.py), taken by lane 0 of the warp that builds the table (stamp_clock):
// the Huffman build stamps row 12 of the chunk, the LL / OF / ML builds rows 13..15 (rows the parse does not use).
B2C_DEV unsigned long long *tables_stamp_row(const ZstdEncParams &P, uint32_t chunk, int row) {
    return P.dbg_cycles ? P.dbg_cycles + ((uint64_t)chunk * 16 + 12 + (uint32_t)row) * 32 : nullptr;
}

B2C_DEV uint32_t chunk_size(const ZstdEncParams &P, uint32_t c) {
    if (P.desc) return P.desc[c].len;
    if (P.src_sizes) return P.src_sizes[c];
    if (P.src_total) {
        const uint64_t off = (uint64_t)c * P.src_stride;
        return (uint32_t)(P.src_total - off < P.src_size_all ? P.src_total - off : P.src_size_all);
    }
    return P.src_size_all;
}
B2C_DEV const uint8_t *chunk_src(const ZstdEncParams &P, uint32_t c) {
    return P.desc ? P.src_base + P.desc[c].off : P.src_base + (uint64_t)c * P.src_stride;
}
B2C_DEV uint32_t chunk_hist(const ZstdEncParams &P, uint32_t c) { return P.desc ? P.desc[c].hist : 0u; }
B2C_DEV uint32_t chunk_last(const ZstdEncParams &P, uint32_t c) { return P.desc ? (P.desc[c].flags & 1u) : 1u; }

// ---- work pool layout (one slab per chunk) ----
B2C_DEV uint32_t wk_off_lit() { return 0; }
B2C_DEV uint32_t wk_off_of(const ZstdEncParams &P) { return (P.blockmax + 64 + 15) & ~15u; }
B2C_DEV uint32_t wk_off_ll(const ZstdEncParams &P) { return wk_off_of(P) + 4 * P.maxseq; }
B2C_DEV uint32_t wk_off_ml(const ZstdEncParams &P) { return wk_off_ll(P) + (P.big ? 4u : 2u) * P.maxseq; }
B2C_DEV uint32_t wk_off_codes(const ZstdEncParams &P) { return wk_off_ml(P) + (P.big ? 4u : 2u) * P.maxseq; }
B2C_DEV uint32_t wk_off_stb(const ZstdEncParams &P) { return wk_off_codes(P) + 3 * P.maxseq; }
B2C_DEV uint8_t *wk_slab(const ZstdEncParams &P, uint32_t chunk) { return P.pool + (uint64_t)chunk * P.pool_stride; }
B2C_DEV uint8_t *wk_lit(const ZstdEncParams &P, uint32_t chunk) { return wk_slab(P, chunk); }
B2C_DEV uint32_t *wk_of(const ZstdEncParams &P, uint32_t chunk) { return reinterpret_cast<uint32_t *>(wk_slab(P, chunk) + wk_off_of(P)); }
B2C_DEV uint8_t *wk_codes(const ZstdEncParams &P, uint32_t chunk, int c) { return wk_slab(P, chunk) + wk_off_codes(P) + (uint32_t)c * P.maxseq; }
B2C_DEV uint16_t *wk_stb(const ZstdEncParams &P, uint32_t chunk, int c) {
    return reinterpret_cast<uint16_t *>(wk_slab(P, chunk) + wk_off_stb(P)) + (uint32_t)c * P.maxseq;
}
// host side of the layout: slab bytes for a block size (maxseq = blockmax / 4 + 64: a match is at least 4 bytes)
static inline uint32_t wk_maxseq(uint32_t blockmax) { return blockmax / 4 + 64; }
static inline uint64_t wk_pool_stride(uint32_t blockmax) {
    const uint64_t ms = wk_maxseq(blockmax), lenb = blockmax > 65536 ? 4 : 2;
    return (((uint64_t)blockmax + 64 + 15) & ~15ull) + 4 * ms + 2 * lenb * ms + 3 * ms + 6 * ms;
}
// The same layout for a block size known at compile time (K4, whose template BLOCK is the launch's blockmax): every
// array sits at a constant offset from the slab.
template <uint32_t BLOCK> struct WkLayout {
    static constexpr uint32_t MAXSEQ = BLOCK / 4 + 64, LENB = BLOCK > 65536 ? 4u : 2u;
    static constexpr uint32_t OF = (BLOCK + 64 + 15) & ~15u, LL = OF + 4 * MAXSEQ, ML = LL + LENB * MAXSEQ;
    static constexpr uint32_t CODES = ML + LENB * MAXSEQ, STB = CODES + 3 * MAXSEQ;
};
// litLen / matchLen-3 of sequence i (u16 arrays for blocks <= 64 KiB, u32 above)
struct WkLens {
    uint8_t *ll, *ml;
    uint32_t big;
    B2C_DEV void put(uint32_t i, uint32_t vll, uint32_t vml) const {
        if (big) { reinterpret_cast<uint32_t *>(ll)[i] = vll; reinterpret_cast<uint32_t *>(ml)[i] = vml; }
        else { reinterpret_cast<uint16_t *>(ll)[i] = (uint16_t)vll; reinterpret_cast<uint16_t *>(ml)[i] = (uint16_t)vml; }
    }
    // plain loads: for values written earlier in the SAME kernel (the read-only path is not coherent with them)
    B2C_DEV uint32_t peek_ll(uint32_t i) const { return big ? reinterpret_cast<const uint32_t *>(ll)[i] : (uint32_t)reinterpret_cast<const uint16_t *>(ll)[i]; }
    B2C_DEV uint32_t peek_ml(uint32_t i) const { return big ? reinterpret_cast<const uint32_t *>(ml)[i] : (uint32_t)reinterpret_cast<const uint16_t *>(ml)[i]; }
    B2C_DEV uint32_t get_ll(uint32_t i) const {
        return big ? B2C_LDG(reinterpret_cast<const uint32_t *>(ll) + i) : (uint32_t)B2C_LDG(reinterpret_cast<const uint16_t *>(ll) + i);
    }
    B2C_DEV uint32_t get_ml(uint32_t i) const {
        return big ? B2C_LDG(reinterpret_cast<const uint32_t *>(ml) + i) : (uint32_t)B2C_LDG(reinterpret_cast<const uint16_t *>(ml) + i);
    }
};
B2C_DEV WkLens wk_lens(const ZstdEncParams &P, uint32_t chunk) {
    WkLens w; w.ll = wk_slab(P, chunk) + wk_off_ll(P); w.ml = wk_slab(P, chunk) + wk_off_ml(P); w.big = P.big; return w;
}

// 6-byte multiplicative hash: two 32-bit multiply-adds (the reference's hashLen(u, bits, 6), zstd/hash.go:27,
// is a 64-bit multiply = ~8 integer instructions per position on the SM; table contents are an
// implementation detail, only the verified matches reach the output).
B2C_DEV uint32_t enc_hash6(uint32_t lo, uint32_t hi) {
    return lo * 0x9E3779B1u + (hi & 0xffffu) * 0x85EBCA6Bu;
}

// length of the common prefix of src[a..limitA) and src[b..], cooperative over the warp
B2C_DEV uint32_t warp_match_len(const uint8_t *src, uint32_t a, uint32_t b, uint32_t limitA) {
    unsigned lane = lane_id();
    uint32_t rem = limitA - a;
    uint32_t k = 0;
    for (;;) {
        uint32_t pos = k + 4 * lane;
        uint32_t eq = 0;
        if (pos < rem) {
            uint32_t x = ld32u(src, a + pos) ^ ld32u(src, b + pos);
            eq = x ? (uint32_t)(__ffs((int)x) - 1) >> 3 : 4u;
            uint32_t nv = rem - pos;
            if (eq > nv) eq = nv;
        }
        unsigned stop = __ballot_sync(FULLMASK, eq < 4);
        if (stop) {
            int fl = __ffs((int)stop) - 1;
            uint32_t e = __shfl_sync(FULLMASK, eq, fl);
            return k + 4 * (uint32_t)fl + e;
        }
        k += 128;
    }
}

struct ParseShared {
    uint32_t ws[40];        // block scan scratch
    uint32_t nextChunk, pad0, kind, rleLen;   // nextChunk: the chunk this CTA takes next (dynamic schedule of the persistent kernels)
    uint64_t mbar;
};
// ------------------------------------------------------------------------------------------------ K1
// ---- S2 / Snappy byte-tag emitters for offsets < 65536 (s2/encode_go.go:80-289; byte layouts pinned by the KATs of
// s2/s2_test.go:827-942).  *_size give the bytes the matching put would write.
enum { LZ_MODE_ZSTD = 0, LZ_MODE_S2 = 1, LZ_MODE_SNAPPY = 2 };

B2C_DEV uint32_t s2_lit_hdr_size(uint32_t ll) { return ll == 0 ? 0u : (ll <= 60 ? 1u : (ll <= 256 ? 2u : 3u)); }
B2C_DEV uint32_t s2_put_lit_hdr(uint8_t *d, uint32_t ll) {   // emitLiteral's tag bytes (ll <= 65536)
    if (ll == 0) return 0;
    const uint32_t n = ll - 1;
    if (n < 60) { d[0] = (uint8_t)(n << 2); return 1; }
    if (n < 256) { d[0] = 60 << 2; d[1] = (uint8_t)n; return 2; }
    d[0] = 61 << 2; d[1] = (uint8_t)n; d[2] = (uint8_t)(n >> 8);
    return 3;
}
B2C_DEV uint32_t s2_repeat_size(uint32_t off, uint32_t len) {
    len -= 4;
    if (len <= 4) return 2;
    if (len < 8 && off < 2048) return 2;
    if (len < (1 << 8) + 4) return 3;
    if (len < (1 << 16) + (1 << 8)) return 4;
    return 5;
}
B2C_DEV uint32_t s2_put_repeat(uint8_t *d, uint32_t off, uint32_t len) {   // emitRepeat, len < 2^16 + 2^8 + 4 here
    len -= 4;
    if (len <= 4) { d[0] = (uint8_t)(len << 2 | 1); d[1] = 0; return 2; }
    if (len < 8 && off < 2048) { d[1] = (uint8_t)off; d[0] = (uint8_t)((off >> 8) << 5 | len << 2 | 1); return 2; }
    if (len < (1 << 8) + 4) { len -= 4; d[2] = (uint8_t)len; d[1] = 0; d[0] = 5 << 2 | 1; return 3; }
    if (len < (1 << 16) + (1 << 8)) { len -= 1 << 8; d[3] = (uint8_t)(len >> 8); d[2] = (uint8_t)len; d[1] = 0; d[0] = 6 << 2 | 1; return 4; }
    len -= 1 << 16;
    d[4] = (uint8_t)(len >> 16); d[3] = (uint8_t)(len >> 8); d[2] = (uint8_t)len; d[1] = 0; d[0] = 7 << 2 | 1;
    return 5;
}
B2C_DEV uint32_t s2_copy_size(uint32_t off, uint32_t len) {
    if (len > 64) return (off < 2048) ? 2 + s2_repeat_size(off, len - 8) : 3 + s2_repeat_size(off, len - 60);
    return (len >= 12 || off >= 2048) ? 3u : 2u;
}
B2C_DEV uint32_t s2_put_copy(uint8_t *d, uint32_t off, uint32_t len) {   // emitCopy, offset < 65536
    if (len > 64) {
        uint32_t o;
        if (off < 2048) { d[1] = (uint8_t)off; d[0] = (uint8_t)((off >> 8) << 5 | (8 - 4) << 2 | 1); len -= 8; o = 2; }
        else { d[2] = (uint8_t)(off >> 8); d[1] = (uint8_t)off; d[0] = 59 << 2 | 2; len -= 60; o = 3; }
        return o + s2_put_repeat(d + o, off, len);
    }
    if (len >= 12 || off >= 2048) { d[2] = (uint8_t)(off >> 8); d[1] = (uint8_t)off; d[0] = (uint8_t)((len - 1) << 2 | 2); return 3; }
    d[1] = (uint8_t)off; d[0] = (uint8_t)((off >> 8) << 5 | (len - 4) << 2 | 1);
    return 2;
}
B2C_DEV uint32_t snappy_copy_size(uint32_t off, uint32_t len) {
    uint32_t sz = 0;
    while (len > 64) { sz += 3; len -= 60; }
    return sz + ((len >= 12 || off >= 2048) ? 3u : 2u);
}
B2C_DEV uint32_t snappy_put_copy(uint8_t *d, uint32_t off, uint32_t len) {   // emitCopyNoRepeat, offset < 65536
    uint32_t o = 0;
    while (len > 64) { d[o + 2] = (uint8_t)(off >> 8); d[o + 1] = (uint8_t)off; d[o] = 59 << 2 | 2; len -= 60; o += 3; }
    if (len >= 12 || off >= 2048) { d[o + 2] = (uint8_t)(off >> 8); d[o + 1] = (uint8_t)off; d[o] = (uint8_t)((len - 1) << 2 | 2); return o + 3; }
    d[o + 1] = (uint8_t)off; d[o] = (uint8_t)((off >> 8) << 5 | (len - 4) << 2 | 1);
    return o + 2;
}

// ------------------------------------------------------------------------------------------------ K2
// Every warp of a K2 CTA builds all four tables of its own chunks, one chunk after another: the Huffman table (rank
// sort, depths, code values, weight normalisation and table fill by all 32 lanes; the tree merge, setMaxHeight's repair
// and the weight encode on lane 0), then the LL, OF and ML tables (normalisation, table fill and size estimates by all
// lanes; the NCount on lane 0).  The warps share only the predefined tables and never wait for each other, so an SM keeps
// one table build in flight per resident warp.
#ifndef TABLES_MIN_CTAS
#define TABLES_MIN_CTAS 5      // resident K2 CTAs per SM the register allocation is held to (44 KB shared memory each)
#endif
constexpr int TABLES_NT = 128;
constexpr int TABLES_NW = TABLES_NT / 32;
struct TablesWarp {
    HufWork hw;
    SeqTableWork st;
};
struct TablesShared {
    SeqWork sw;                 // the predefined tables
    TablesWarp wk[TABLES_NW];
};
B2C_DEV void zstd_tables_chunk(const SeqWork *sw, TablesWarp *tw, const ZstdEncParams &P, uint32_t chunk) {
    const unsigned lane = threadIdx.x & 31;
    ChunkWork *W = P.work + chunk;
    if (W->kind != 0) return;
    const uint32_t nseq = W->nseq, nlit = W->nlit;
    {
        HufWork *hw = &tw->hw;
        unsigned long long *hrow = tables_stamp_row(P, chunk, 0);
        for (uint32_t s = lane; s < 256; s += 32) hw->count[s] = W->litHist[s];
        if (lane == 0) { hw->status = HUF_INCOMPRESSIBLE; hw->tableDescLen = 0; hw->tableLog = 0; }
        __syncwarp();
        stamp_clock(hrow, 0);
        if (nlit > 16) {
            huf_bt_stats(hw, nlit, lane);
            __syncwarp();
            if (hw->status == HUF_OK) {
                huf_bt_sort(hw, lane, 32);
                __syncwarp();
                stamp_clock(hrow, 1);
                if (lane == 0) huf_bt_merge(hw);
                __syncwarp();
                stamp_clock(hrow, 2);
                huf_bt_depths(hw, lane);
                stamp_clock(hrow, 3);
                huf_bt_ranks(hw, nlit, lane);
                stamp_clock(hrow, 4);
                huf_bt_bits(hw, lane, 32);
                __syncwarp();
                huf_bt_vals(hw, lane, 32);
                __syncwarp();
                stamp_clock(hrow, 5);
                huf_bt_write(hw, lane);
                stamp_clock(hrow, 6);
            }
        }
        if (hw->status == HUF_OK) {
            for (uint32_t s = lane; s < 256; s += 32) { W->ctVal[s] = hw->ctVal[s]; W->ctBits[s] = hw->ctBits[s]; }
            for (uint32_t i = lane; i < hw->tableDescLen; i += 32) W->tableDesc[i] = hw->tableDesc[i];
        }
        if (lane == 0) { W->hufStatus = (uint32_t)hw->status; W->hufTableLog = hw->tableLog; W->tableDescLen = hw->tableDescLen; }
        stamp_clock(hrow, 7);
    }
    for (int which = 0; which < 3; which++) {
        SeqTableWork *st = &tw->st;
        unsigned long long *srow = tables_stamp_row(P, chunk, 1 + which);
        for (uint32_t s = lane; s < 64; s += 32) st->hist[s] = W->seqHist[which][s];
        __syncwarp();
        seq_build_table(st, &sw->predef[which], W->maxSym[which] + 1, nseq, wk_codes(P, chunk, which)[0], lane, srow);
        // publish the table this chain will use
        const FseCTable *t = st->used ? &st->cur : &sw->predef[which];
        const uint32_t *s32 = reinterpret_cast<const uint32_t *>(t);
        uint32_t *d32 = reinterpret_cast<uint32_t *>(&W->tbl[which]);
        for (uint32_t i = lane; i < sizeof(FseCTable) / 4; i += 32) d32[i] = s32[i];
        for (uint32_t i = lane; i < st->ncountLen && i < 96; i += 32) W->ncount[which][i] = st->ncount[i];
        if (lane == 0) {
            W->mode[which] = st->mode; W->ncountLen[which] = st->ncountLen;
            if (st->ncountLen == SEQ_TABLE_ERR) { W->ncountLen[which] = 0; W->kind = 1; }  // internal error: store raw
        }
        __syncwarp();
        stamp_clock(srow, 5);
    }
}

// The chunk loop of a K2 CTA: warp w takes chunks first * TABLES_NW + w, then every stride * TABLES_NW-th one.
B2C_DEV void zstd_tables_loop(TablesShared *ts, const ZstdEncParams &P, uint32_t first, uint32_t stride) {
    const unsigned w = threadIdx.x >> 5;
    for (uint32_t c = first * TABLES_NW + w; c < P.nchunks; c += stride * TABLES_NW) zstd_tables_chunk(&ts->sw, &ts->wk[w], P, c);
}

// ------------------------------------------------------------------------------------------------ K3
// One lane per (chunk, chain): CTA = 96 threads = 3 warps; warp c walks chain c of 32 consecutive chunks.
// Per-lane tables live in shared memory, interleaved so that lane l only ever touches bank l:
// 128 words of packed u16 next-states + 64 words of (deltaNbBits | (deltaFindState + 512) << 21).
constexpr int CHAIN_NT = 96;
constexpr int CHAIN_XXH_NT = 128;   // optional extra warps of a chains CTA: XXH64 of its 32 chunks, four lanes per chunk
constexpr uint32_t CHAIN_SMEM_WORDS_PER_LANE = 64 + 56;   // 256 x u8 next-state offsets + 56 x u32 symbol transforms
constexpr uint32_t CHAIN_SMEM_BYTES = CHAIN_NT * CHAIN_SMEM_WORDS_PER_LANE * 4;
// K3: one lane per (chunk, table) walks the tANS state chain from the last sequence to the first
// (blockenc.go:757-803 restated as three independent recurrences) and stores, per sequence, the bits it emits:
// stb[i] = value | nbBits << 12.  The recurrence is latency-bound, so the loop keeps the dependent path to
// add/shift/add + one shared-memory load per step: codes arrive eight at a time (one 8-byte load, requested two
// blocks ahead), their symbol transforms are fetched up front, results leave as one 16-byte store per 8 steps.
// Per-lane tables are interleaved so lane l only touches bank l: next states are kept as u8 offsets from tableSize
// (4 per word), 45 KB per CTA, so five CTAs fit an SM and a 16 384-chunk batch is a single wave.
B2C_DEV void zstd_chains_block(uint32_t *smem32, const ZstdEncParams &P, uint32_t chunk0) {
    const unsigned tid = threadIdx.x, lane = tid & 31, which = tid >> 5;
    const uint32_t chunk = chunk0 + lane;
    const bool live = chunk < P.nchunks && P.work[chunk < P.nchunks ? chunk : 0].kind == 0;
    ChunkWork *W = P.work + (live ? chunk : 0);
    uint32_t *st32 = smem32 + which * 32 * CHAIN_SMEM_WORDS_PER_LANE;  // this warp's region
    uint8_t *tState = reinterpret_cast<uint8_t *>(st32 + lane);        // element i at byte (i >> 2) * 128 + (i & 3)
    uint32_t *tSym = st32 + 64 * 32 + lane;                            // element i of lane l at word i * 32 + l
#define TSTATE(i) tState[(((uint32_t)(i)) >> 2) * 128 + (((uint32_t)(i)) & 3)]
    uint32_t nseq = 0, useRLE = 1, tableLog = 0, tableSize = 1;
    if (live) {
        const FseCTable *t = &W->tbl[which];
        nseq = W->nseq; useRLE = t->useRLE; tableLog = t->tableLog; tableSize = 1u << tableLog;
        if (!useRLE) {
            const uint32_t *sw = reinterpret_cast<const uint32_t *>(t->stateTable);
            const uint32_t ts2 = tableSize / 2;
            for (uint32_t i = 0; i < ts2; i += 2) {      // tableSize >= 32: four states per word
                const uint32_t v0 = sw[i], v1 = sw[i + 1];
                st32[(i >> 1) * 32 + lane] = ((v0 & 0xffff) - tableSize) | (((v0 >> 16) - tableSize) << 8) |
                                             (((v1 & 0xffff) - tableSize) << 16) | (((v1 >> 16) - tableSize) << 24);
            }
            const uint32_t sl = t->symbolLen;
            for (uint32_t i = 0; i < 56; i++)
                tSym[i * 32] = (i < sl) ? (t->deltaNbBits[i] | ((uint32_t)((int32_t)t->deltaFindState[i] + 512) << 21)) : 0u;
        }
    }
    __syncwarp();
    const uint8_t *codes = wk_codes(P, live ? chunk : 0, (int)which);
    uint16_t *stb = wk_stb(P, live ? chunk : 0, (int)which);
    uint32_t state = 0;
    const bool run = live && !useRLE && nseq >= 1;
    if (run) {
        const uint32_t e = tSym[(codes[nseq - 1] < 56u ? codes[nseq - 1] : 0u) * 32];
        const uint32_t dnb = e & 0x1fffffu;
        const int32_t dfs = (int32_t)(e >> 21) - 512;
        const uint32_t nbBitsOut = (dnb + (1u << 15)) >> 16;
        const int32_t im = (int32_t)((nbBitsOut << 16) - dnb);
        state = tableSize + TSTATE((im >> nbBitsOut) + dfs);
    }
    // sequences nseq-2 .. 0 in blocks of eight (block k = sequences 8k .. 8k+7), top block first
    const int32_t top = run ? (int32_t)nseq - 2 : -1;
    const int32_t blk = top >> 3;                                  // -1 when there is nothing to do
    const uint32_t nblk = warp_max((uint32_t)(blk + 1));
    const uint2 *c8 = reinterpret_cast<const uint2 *>(codes);
    uint2 cwA = make_uint2(0, 0), cwB = make_uint2(0, 0);
    if (blk >= 0) cwA = c8[blk];
    if (blk >= 1) cwB = c8[blk - 1];
    for (uint32_t it = 0; it < nblk; it++) {
        const int32_t k = blk - (int32_t)it;
        if (k >= 0) {
            uint2 cwC = make_uint2(0, 0);
            if (k >= 2) cwC = c8[k - 2];
            uint32_t e[8];
#pragma unroll
            for (int j = 0; j < 8; j++) {
                uint32_t code = (((j < 4) ? cwA.x : cwA.y) >> (8 * (j & 3))) & 63u;
                if (code >= 56u) code = 0;     // bytes past the last sequence are not codes
                e[j] = tSym[code * 32];
            }
            uint32_t o[4] = {0, 0, 0, 0};
#pragma unroll
            for (int pos = 7; pos >= 0; pos--) {
                if (8 * k + pos <= top) {
                    const uint32_t nb = (state + (e[pos] & 0x1fffffu)) >> 16;
                    o[pos >> 1] |= ((state & ((1u << nb) - 1)) | (nb << 12)) << (16 * (pos & 1));
                    state = tableSize + TSTATE((int32_t)(state >> nb) + (int32_t)(e[pos] >> 21) - 512);
                }
            }
            *reinterpret_cast<uint4 *>(stb + 8 * k) = make_uint4(o[0], o[1], o[2], o[3]);
            cwA = cwB; cwB = cwC;
        }
    }
    if (live) {
        if (useRLE) { for (uint32_t i = 0; i + 1 < nseq; i++) stb[i] = 0; state = 0; }
        W->finalState[which] = state;
    }
#undef TSTATE
}

// ------------------------------------------------------------------------------------------------ K4
struct PackShared {
    HufWork hw;               // only ctVal/ctBits/tableDesc*/scan/stream* hold their usual content here; two unused
                              // members are reused (two CTAs must fit an SM, there is no kilobyte to spare):
                              //   hw.count[256] = Huffman codes as (code | nbits << 16)               (PACK_PK)
                              //   hw.nsym[0..127] = extra-bit counts per LL / ML code, seqenc.go:61-97  (PACK_LLB / PACK_MLB)
    uint32_t scan[40];
    uint32_t litMode, lhSize, litPayload, seqOff, total, blockBytes, nc0, nc1;   // the byte phase's layout
    uint64_t mbar;            // completion of the literals' bulk copy
};
#if PACK_BITS_LUT
#define PACK_LLB(c) ((uint32_t)ps->hw.nsym[(c) & 63])
#define PACK_MLB(c) ((uint32_t)ps->hw.nsym[64 + ((c) & 63)])
#else
#define PACK_LLB(c) seq_ll_bits(c)
#define PACK_MLB(c) seq_ml_bits(c)
#endif
#ifndef PACK_LIT_SMEM_BYTES
#define PACK_LIT_SMEM_BYTES (40 * 1024)
#endif
// K4 shared-memory plan per block size: the staging buffer holds the whole output, literals are staged when they fit.
// 64 KiB blocks: 64 K + 40 K -> two CTAs per SM; 128 KiB blocks (level 2): 128 K + 64 K -> one CTA per SM.
template <uint32_t BLOCK> struct PackCfg {
    static constexpr uint32_t STAGE_BYTES = BLOCK + 128;
    static constexpr uint32_t LIT_SMEM = (BLOCK <= 65536) ? (uint32_t)PACK_LIT_SMEM_BYTES : 64u * 1024u;
    static constexpr uint32_t SMEM_SH = STAGE_BYTES + LIT_SMEM;
    static constexpr uint32_t SMEM_BYTES = SMEM_SH + ((sizeof(PackShared) + 15) / 16) * 16;
};
constexpr uint32_t PACK_SMEM_BYTES = PackCfg<65536>::SMEM_BYTES;
static_assert(PACK_LIT_SMEM_BYTES != 40 * 1024 || 2 * (PACK_SMEM_BYTES + 1024) <= 228 * 1024, "two K4 CTAs must fit one SM");
static_assert(PackCfg<131072>::SMEM_BYTES <= 227 * 1024, "the 128 KiB K4 CTA must fit one SM");

B2C_DEV uint32_t frame_header_bytes(uint32_t n) {
    if (n == 0) return 6;
    bool single = n > 1024;
    uint32_t fh = 4 + 1 + (single ? 0 : 1);
    if (n >= 256) fh += (n >= 65536 + 256) ? 4 : 2; else if (single) fh += 1;
    return fh;
}
// frameHeader.appendTo (frameenc.go:25-92), single chunk, no dictionary
B2C_DEV uint32_t write_frame_header(uint8_t *o8, uint32_t n, bool crc) {
    uint32_t o = 0;
    o8[o++] = 0x28; o8[o++] = 0xB5; o8[o++] = 0x2F; o8[o++] = 0xFD;
    if (n == 0) { o8[o++] = 32; o8[o++] = 0; return o; }  // WithZeroFrames (encoder.go:732-751)
    bool single = n > 1024;
    uint32_t fcs = (n >= 256) ? ((n >= 65536 + 256) ? 2u : 1u) : 0u;
    o8[o++] = (uint8_t)((crc ? 4u : 0u) | (single ? 32u : 0u) | (fcs << 6));
    if (!single) {
        uint32_t ws = 1u << (32 - (uint32_t)__clz((int)n));  // WindowSize(n) (enc_base.go:42-50)
        if (ws < 1024) ws = 1024;
        o8[o++] = (uint8_t)(((32 - (uint32_t)__clz((int)(ws - 1))) - 10) << 3);
    }
    if (fcs == 0) { if (single) o8[o++] = (uint8_t)n; }
    else if (fcs == 1) { uint32_t v = n - 256; o8[o++] = (uint8_t)v; o8[o++] = (uint8_t)(v >> 8); }
    else { o8[o++] = (uint8_t)n; o8[o++] = (uint8_t)(n >> 8); o8[o++] = (uint8_t)(n >> 16); o8[o++] = (uint8_t)(n >> 24); }
    return o;
}

// huff0 compress(): out >= wantSize => ErrIncompressible (compress.go:155-158, WantLogLess 4), then blockenc.go:534-544:
// the literals' mode, 0 raw, 1 RLE, 2 compressed (payload: Huffman bytes, meaningful when the table was built)
B2C_DEV uint32_t lit_mode(int32_t hufStatus, uint32_t payload, uint32_t nlit) {
    if (hufStatus != HUF_OK) return (hufStatus == HUF_USE_RLE) ? 1u : 0u;
    if (payload >= nlit - (nlit >> 4)) return 0;
    if (payload + 5 > nlit) {
        // compare with the raw representation
        const uint32_t inBits = 32 - (uint32_t)__clz((int)nlit);
        const uint32_t szRaw = inBits < 5 ? 1 : (inBits < 12 ? 2 : 3);
        const uint32_t compBits = payload ? 32 - (uint32_t)__clz((int)payload) : 0;
        const uint32_t szComp = (compBits <= 10 && inBits <= 10) ? 3 : ((compBits <= 14 && inBits <= 14) ? 4 : 5);
        if (payload + szComp >= nlit + szRaw) return 0;
    }
    return 2;
}
// bytes of the literals section header (blockenc.go:153-238)
B2C_DEV uint32_t lit_header_bytes(uint32_t mode, uint32_t payload, uint32_t nlit) {
    if (mode == 2) {
        const uint32_t inBits = 32 - (uint32_t)__clz((int)nlit);
        const uint32_t compBits = payload ? 32 - (uint32_t)__clz((int)payload) : 0;
        return (compBits <= 10 && inBits <= 10) ? 3 : ((compBits <= 14 && inBits <= 14) ? 4 : 5);
    }
    const uint32_t inBits = nlit ? 32 - (uint32_t)__clz((int)nlit) : 0;
    return inBits < 5 ? 1 : (inBits < 12 ? 2 : 3);
}
// the literals section header, little-endian in its lhSize low bytes
B2C_DEV uint64_t lit_header(uint32_t mode, uint32_t lhSize, uint32_t nlit, uint32_t payload, bool four) {
    if (mode == 2) {
        const uint64_t comp = payload;
        if (lhSize == 3) return 2u | ((four ? 1u : 0u) << 2) | ((uint64_t)nlit << 4) | (comp << 14);
        if (lhSize == 4) return 2u | (2u << 2) | ((uint64_t)nlit << 4) | (comp << 18);
        return 2u | (3u << 2) | ((uint64_t)nlit << 4) | (comp << 22);
    }
    const uint64_t ty = (mode == 1) ? 1u : 0u;
    if (lhSize == 1) return ty | ((uint64_t)nlit << 3);
    if (lhSize == 2) return ty | (1u << 2) | ((uint64_t)nlit << 4);
    return ty | (3u << 2) | ((uint64_t)nlit << 4);
}
// element j (a compile-time constant after unrolling) of eight u8 / u16 / u32 values loaded together
B2C_DEV uint32_t u8_of(uint2 v, int j) { return ((j < 4 ? v.x : v.y) >> (8 * (j & 3))) & 255u; }
B2C_DEV uint32_t u16_of(uint4 v, int j) {
    const uint32_t w = j < 2 ? v.x : (j < 4 ? v.y : (j < 6 ? v.z : v.w));
    return (w >> (16 * (j & 1))) & 0xffffu;
}
B2C_DEV uint32_t u32_of(uint4 a, uint4 b, int j) {
    const uint4 v = j < 4 ? a : b;
    return (j & 3) == 0 ? v.x : ((j & 3) == 1 ? v.y : ((j & 3) == 2 ? v.z : v.w));
}

// K4, one CTA per chunk.  Barriers: the sequence scan (2), the Huffman sizes (5, shared with huff0), the end of the
// word-granular phase and the end of the byte-granular phase.
//   top      literals into shared memory by one bulk copy (waited for where they are first read); the Huffman table,
//            the per-chunk scalars and the first sequences' codes and state bits requested together; stage zeroed
//   seq size thread t owns a contiguous run of 8-aligned groups of sequences (thread 0 the top ones: the bitstream runs
//            from the last sequence to the first); each group is one 8-byte load per code table and one 16-byte
//            load per state-bit table, its lengths and offsets are prefetched into L2 for the pack pass; block scan
//   huf size code-length sums and their scan (huf_enc_sizes); every thread then derives the literal mode and all offsets
//   words    the Huffman streams and the sequence bitstream, each thread its own bit range of the zeroed stage
//   bytes    frame / block / literals / sequences headers, NCount bytes, the table description, raw or RLE literals,
//            the checksum, each field by its own thread
//   write-back, one coalesced copy (raw / RLE blocks skip the stage)
template <uint32_t BLOCK>
B2C_DEV void zstd_pack_chunk(uint8_t *smem, const ZstdEncParams &P, uint32_t chunk) {
    constexpr uint32_t PACK_STAGE_BYTES = PackCfg<BLOCK>::STAGE_BYTES;
    constexpr uint32_t PACK_LIT_SMEM = PackCfg<BLOCK>::LIT_SMEM;
    constexpr bool BIG = BLOCK > 65536;   // litLen / matchLen arrays are u32 (P.big)
    const unsigned tid = threadIdx.x;
    uint8_t *stage = smem;
    PackShared *ps = reinterpret_cast<PackShared *>(smem + PackCfg<BLOCK>::SMEM_SH);
    ChunkWork *W = P.work + chunk;
    uint8_t *gdst = P.dst_base + (uint64_t)chunk * P.dst_stride;
    const uint32_t n = W->n;
    const uint32_t lastBit = chunk_last(P, chunk);
    const bool frame = (P.flags & ENC_FLAG_FRAME) != 0;
    const bool crc = frame && (P.flags & ENC_FLAG_CRC) != 0;
    uint32_t kind = W->kind;
    if (kind == 3) { if (tid == 0) P.out_sizes[chunk] = -3; return; }
    const uint32_t nseq = W->nseq, nlit = W->nlit;
    const uint32_t fh = frame ? frame_header_bytes(n) : 0;
    B2C_PACK_PHASE(0);

    if (kind == 0) {
        // ------------------------------------------------------------ literals: one bulk copy into shared memory
        using L = WkLayout<BLOCK>;
        const uint8_t *slab = wk_slab(P, chunk);
        const uint8_t *lit = slab;
        uint8_t *ls = smem + PACK_STAGE_BYTES;
        const bool litSmem = nlit <= PACK_LIT_SMEM;
#ifndef B2C_EMU
        // rounded up to 16 bytes: the slab's literal area has 64 bytes behind the largest block
        const bool bulk = litSmem && nlit > 0 && (reinterpret_cast<uintptr_t>(lit) & 15) == 0;
        if (bulk && tid == 0) {
            mbar_init(&ps->mbar, 1);
            mbar_fence_init();
            mbar_expect_tx(&ps->mbar, (nlit + 15) & ~15u);
            tma_load_1d(ls, lit, (nlit + 15) & ~15u, &ps->mbar);
        }
#else
        const bool bulk = false;
#endif
        if (litSmem && !bulk) {   // ordered before the first read by the sequence scan's barriers
            if ((reinterpret_cast<uintptr_t>(lit) & 15) == 0) {
                const uint4 *g4 = reinterpret_cast<const uint4 *>(lit);
                for (uint32_t i = tid; i < (nlit + 15) / 16; i += PACK_NT) reinterpret_cast<uint4 *>(ls)[i] = g4[i];
            } else {
                for (uint32_t i = tid; i < nlit; i += PACK_NT) ls[i] = lit[i];
            }
        }
        // ------------------------------------------------------------ requests: Huffman table, chunk scalars
        HufWork *hw = &ps->hw;
        uint32_t ctv = 0, ctb = 0, tdb = 0;
        if (tid < 256) { ctv = W->ctVal[tid]; ctb = W->ctBits[tid]; }
        if (tid < 320) tdb = W->tableDesc[tid];   // all 320 bytes: no wait for tableDescLen
        const int32_t hufStatus = (int32_t)W->hufStatus;
        const uint32_t tableDescLen = W->tableDescLen;
        const uint32_t nc0 = W->ncountLen[0], nc1 = W->ncountLen[1], ncSum = nc0 + nc1 + W->ncountLen[2];
        const uint32_t tlLL = W->tbl[TBL_LL].tableLog, tlOF = W->tbl[TBL_OF].tableLog, tlML = W->tbl[TBL_ML].tableLog;
        // the stage holds the output; zero every word a bit writer may OR into.  A compressed block is smaller than the
        // chunk (else it is stored raw), so everything it writes lies below fh + 3 + n + 4.
        {
            const uint32_t zb = fh + 3 + n + 4 + 8;
            const uint32_t z16 = (zb < PACK_STAGE_BYTES ? zb + 15 : PACK_STAGE_BYTES) / 16;
            for (uint32_t i = tid; i < z16; i += PACK_NT) reinterpret_cast<uint4 *>(stage)[i] = make_uint4(0, 0, 0, 0);
        }
        B2C_PACK_PHASE(5);

        // ------------------------------------------------------------ sequence bitstream sizes
        const uint2 *cLL = reinterpret_cast<const uint2 *>(slab + L::CODES + TBL_LL * L::MAXSEQ);
        const uint2 *cOF = reinterpret_cast<const uint2 *>(slab + L::CODES + TBL_OF * L::MAXSEQ);
        const uint2 *cML = reinterpret_cast<const uint2 *>(slab + L::CODES + TBL_ML * L::MAXSEQ);
        const uint4 *stbLL = reinterpret_cast<const uint4 *>(slab + L::STB + 2 * TBL_LL * L::MAXSEQ);
        const uint4 *stbOF = reinterpret_cast<const uint4 *>(slab + L::STB + 2 * TBL_OF * L::MAXSEQ);
        const uint4 *stbML = reinterpret_cast<const uint4 *>(slab + L::STB + 2 * TBL_ML * L::MAXSEQ);
        const uint4 *wll = reinterpret_cast<const uint4 *>(slab + L::LL), *wml = reinterpret_cast<const uint4 *>(slab + L::ML);
        const uint4 *wof = reinterpret_cast<const uint4 *>(slab + L::OF);
        // groups of eight sequences [gLo, gHi); entries past nseq are read (the arrays hold maxseq, a multiple of 16)
        // and ignored, and sequence nseq-1 has no state bits (its states start the chains)
        const uint32_t ngrp = (nseq + 7) >> 3, gper = (ngrp + PACK_NT - 1) / PACK_NT;
        const uint32_t gHi = ngrp > tid * gper ? ngrp - tid * gper : 0u, gLo = gHi > gper ? gHi - gper : 0u;
        uint32_t mybits = 0;
        for (uint32_t g = gLo; g < gHi; g++) {
            const uint2 cl8 = B2C_LDG(cLL + g);
            const uint2 co8 = B2C_LDG(cOF + g);
            const uint2 cm8 = B2C_LDG(cML + g);
            const uint4 sl8 = B2C_LDG(stbLL + g);
            const uint4 so8 = B2C_LDG(stbOF + g);
            const uint4 sm8 = B2C_LDG(stbML + g);
            prefetch_l2(wof + 2 * g);
            prefetch_l2(wll + (BIG ? 2 : 1) * g);
            prefetch_l2(wml + (BIG ? 2 : 1) * g);
#pragma unroll
            for (int j = 0; j < 8; j++) {
                const uint32_t idx = 8 * g + j;
                uint32_t b = seq_ll_bits(u8_of(cl8, j)) + seq_ml_bits(u8_of(cm8, j)) + u8_of(co8, j);
                if (idx + 1 < nseq) b += (u16_of(sl8, j) >> 12) + (u16_of(so8, j) >> 12) + (u16_of(sm8, j) >> 12);
                if (idx < nseq) mybits += b;
            }
        }
        if (tid < 256) { hw->ctVal[tid] = (uint16_t)ctv; hw->ctBits[tid] = (uint8_t)ctb; }
        if (tid < 320) hw->tableDesc[tid] = (uint8_t)tdb;
        if (tid < 64) { ps->hw.nsym[tid] = (uint8_t)seq_ll_bits(tid); ps->hw.nsym[64 + tid] = (uint8_t)seq_ml_bits(tid); }
        if (tid == 0) hw->tableDescLen = tableDescLen;
        uint32_t totalBits;
        const uint32_t exBits = group_scan_excl(mybits, ps->scan, 0, PACK_NT, tid, &totalBits);   // also publishes the table
        B2C_PACK_PHASE(4);

        // ------------------------------------------------------------ literals section sizes
#ifndef B2C_EMU
        if (bulk) mbar_wait(&ps->mbar, 0);
#endif
        if (litSmem) lit = ls;
        B2C_PACK_PHASE(1);
        const bool four = nlit >= 1024;
        HufEncState hst;
        uint32_t payload = 0;
        if (hufStatus == HUF_OK) payload = huf_enc_sizes(hw, ps->hw.count, lit, nlit, four ? 1 : 0, tid, PACK_NT, 0, &hst);
        B2C_PACK_PHASE(2);
        // every thread derives the layout; the byte phase reads it back from shared memory, so it is not held in
        // registers across the bit writers
        const uint32_t nsHdr = (nseq < 128) ? 1u : (nseq < 0x7f00 ? 2u : 3u);
        uint32_t litOff, bsStart;   // staging offset of the literal payload, first bit of the sequence bitstream
        bool hufBits, useRaw;
        {
            const uint32_t litMode = lit_mode(hufStatus, payload, nlit), lhSize = lit_header_bytes(litMode, payload, nlit);
            const uint32_t litBytes = (litMode == 2) ? payload : (litMode == 1 ? 1u : nlit);
            litOff = fh + 3 + lhSize;
            const uint32_t seqOff = litOff + litBytes;
            const uint32_t bsOff = seqOff + nsHdr + 1 + ncSum;
            const uint32_t bsBytes = (totalBits + tlML + tlOF + tlLL + 1 + 7) >> 3;
            const uint32_t blockBytes = (bsOff - fh - 3) + bsBytes;  // block content size
            const uint32_t total = fh + 3 + blockBytes + (crc ? 4u : 0u);
            // blockenc.go:811-817: not smaller than the input => raw block.  Also covers staging overflow.
            useRaw = (blockBytes >= n) || (total + 8 > PACK_STAGE_BYTES);
            hufBits = litMode == 2;
            bsStart = bsOff * 8 + exBits;
            if (tid == 0) {
                ps->litMode = litMode; ps->lhSize = lhSize; ps->litPayload = payload; ps->seqOff = seqOff;
                ps->total = total; ps->blockBytes = blockBytes; ps->nc0 = nc0; ps->nc1 = nc1;
            }
        }
        if (!useRaw) {
            // ------------------------------------------------------------ word-granular phase: the two bitstreams
            if (hufBits) huf_enc_pack_bits(ps->hw.count, lit, stage, litOff, &hst);
            B2C_PACK_PHASE(6);
            {
                BitRun br;
                br.init(reinterpret_cast<uint32_t *>(stage), bsStart);
                for (uint32_t g = gHi; g-- > gLo;) {
                    const uint2 cl8 = B2C_LDG(cLL + g);
                    const uint2 co8 = B2C_LDG(cOF + g);
                    const uint2 cm8 = B2C_LDG(cML + g);
                    const uint4 sl8 = B2C_LDG(stbLL + g);
                    const uint4 so8 = B2C_LDG(stbOF + g);
                    const uint4 sm8 = B2C_LDG(stbML + g);
                    const uint4 of0 = B2C_LDG(wof + 2 * g), of1 = B2C_LDG(wof + 2 * g + 1);
                    uint4 ll0, ll1, ml0, ml1;
                    if (BIG) {
                        ll0 = B2C_LDG(wll + 2 * g); ll1 = B2C_LDG(wll + 2 * g + 1);
                        ml0 = B2C_LDG(wml + 2 * g); ml1 = B2C_LDG(wml + 2 * g + 1);
                    } else {
                        ll0 = B2C_LDG(wll + g); ml0 = B2C_LDG(wml + g);
                        ll1 = ml1 = make_uint4(0, 0, 0, 0);
                    }
#pragma unroll
                    for (int j = 7; j >= 0; j--) {
                        const uint32_t idx = 8 * g + j;
                        if (idx < nseq) {
                            const uint32_t cl = u8_of(cl8, j), co = u8_of(co8, j), cm = u8_of(cm8, j);
                            const uint32_t vLL = BIG ? u32_of(ll0, ll1, j) : u16_of(ll0, j);
                            const uint32_t vML = BIG ? u32_of(ml0, ml1, j) : u16_of(ml0, j);
                            const uint32_t vOF = u32_of(of0, of1, j);
                            if (idx + 1 < nseq) {
                                // three state flushes (<= 9 bits each) in one append: OF, ML, LL (blockenc.go:757-790)
                                const uint32_t so = u16_of(so8, j), sm = u16_of(sm8, j), sl = u16_of(sl8, j);
                                const uint32_t no = so >> 12, nm = sm >> 12;
                                br.add((so & 0xfff) | ((sm & 0xfff) << no) | ((sl & 0xfff) << (no + nm)), no + nm + (sl >> 12));
                            }
                            // extra bits: LL and ML (<= 16 bits each) together, then OF
                            const uint32_t lb = PACK_LLB(cl), mb = PACK_MLB(cm);
                            br.add((vLL & ((1u << lb) - 1)) | ((vML & ((1u << mb) - 1)) << lb), lb + mb);
                            br.add(vOF & ((1u << co) - 1), co);
                        }
                    }
                }
                if (gLo == 0 && gHi > 0) {
                    // final states: ml, of, ll (blockenc.go:804-806) + end mark
                    br.add(W->finalState[TBL_ML] & ((1u << tlML) - 1), tlML);
                    br.add(W->finalState[TBL_OF] & ((1u << tlOF) - 1), tlOF);
                    br.add(W->finalState[TBL_LL] & ((1u << tlLL) - 1), tlLL);
                    br.add(1u, 1);
                }
                br.finish();
            }
            __syncthreads();  // byte stores below must not race the word atomics above
            B2C_PACK_PHASE(7);
            // ------------------------------------------------------------ byte-granular phase: one field per thread
            const uint32_t litMode = ps->litMode, lhSize = ps->lhSize, payload = ps->litPayload, seqOff = ps->seqOff;
            const uint32_t total = ps->total, blockBytes = ps->blockBytes, nc0 = ps->nc0, nc1 = ps->nc1;
            const uint32_t tblOff = seqOff + nsHdr + 1, ncSum = nc0 + nc1 + W->ncountLen[2];
            if (tid == 0 && frame) write_frame_header(stage, n, crc);
            if (tid == 32) {
                const uint32_t bh = lastBit | (2u << 1) | (blockBytes << 3);  // compressed block
                stage[fh] = (uint8_t)bh; stage[fh + 1] = (uint8_t)(bh >> 8); stage[fh + 2] = (uint8_t)(bh >> 16);
            }
            if (tid == 64) {
                const uint64_t lh = lit_header(litMode, lhSize, nlit, payload, four);
                for (uint32_t k = 0; k < lhSize; k++) stage[fh + 3 + k] = (uint8_t)(lh >> (8 * k));
            }
            if (tid == 96) {
                uint32_t o = seqOff;
                if (nseq < 128) stage[o++] = (uint8_t)nseq;
                else if (nseq < 0x7f00) { stage[o++] = (uint8_t)(128 + (nseq >> 8)); stage[o++] = (uint8_t)nseq; }
                else { uint32_t v = nseq - 0x7f00; stage[o++] = 255; stage[o++] = (uint8_t)v; stage[o++] = (uint8_t)(v >> 8); }
                stage[o] = (uint8_t)((W->mode[TBL_LL] << 6) | (W->mode[TBL_OF] << 4) | (W->mode[TBL_ML] << 2));
            }
            if (crc && tid >= 128 && tid < 132) stage[total - 4 + (tid - 128)] = (uint8_t)((uint32_t)W->xxh >> (8 * (tid - 128)));
            for (uint32_t k = tid; k < ncSum; k += PACK_NT) {
                const uint32_t c = k < nc0 ? 0u : (k < nc0 + nc1 ? 1u : 2u);
                stage[tblOff + k] = W->ncount[c][k - (c == 0 ? 0u : (c == 1 ? nc0 : nc0 + nc1))];
            }
            if (litMode == 2) huf_enc_pack_header(hw, four, stage, litOff, tid, PACK_NT);
            else if (litMode == 0) { for (uint32_t i = tid; i < nlit; i += PACK_NT) stage[litOff + i] = lit[i]; }
            else if (tid == 0) stage[litOff] = lit[0];
            __syncthreads();
            B2C_PACK_PHASE(8);
            // one coalesced write-back
            if (total <= P.dst_cap) {
                if ((reinterpret_cast<uintptr_t>(gdst) & 15) == 0) {
                    const uint4 *s4 = reinterpret_cast<const uint4 *>(stage);
                    uint4 *d4 = reinterpret_cast<uint4 *>(gdst);
                    uint32_t n16 = total / 16;
                    for (uint32_t i = tid; i < n16; i += PACK_NT) d4[i] = s4[i];
                    for (uint32_t i = n16 * 16 + tid; i < total; i += PACK_NT) gdst[i] = stage[i];
                } else {
                    for (uint32_t i = tid; i < total; i += PACK_NT) gdst[i] = stage[i];
                }
                if (tid == 0) P.out_sizes[chunk] = (int64_t)total;
            } else if (tid == 0) P.out_sizes[chunk] = -4;  // destination too small
            B2C_PACK_PHASE(9);
            if (P.dbg_hdr && tid == 0) {
                uint32_t *d = P.dbg_hdr + (uint64_t)chunk * 4;
                d[0] = nseq; d[1] = nlit; d[2] = 0; d[3] = litMode;
            }
            return;
        }
        kind = 1;  // fall through to the raw block (the bulk copy has landed: every thread waited for it)
    }

    // ---------------------------------------------------------------- raw / RLE block (+ frame), straight to global memory
    {
        const uint32_t hlen = fh + 3;
        const uint32_t body = (kind == 2) ? 1u : n;
        const bool crcHere = crc && n > 0;
        const uint32_t total = hlen + body + (crcHere ? 4u : 0u);
        if (total <= P.dst_cap) {
            if (tid == 0) {
                if (frame) write_frame_header(gdst, n, crc);
                const uint32_t bh = (kind == 2) ? (lastBit | (1u << 1) | (W->rleLen << 3)) : (lastBit | (0u << 1) | (n << 3));
                gdst[fh] = (uint8_t)bh; gdst[fh + 1] = (uint8_t)(bh >> 8); gdst[fh + 2] = (uint8_t)(bh >> 16);
                P.out_sizes[chunk] = (int64_t)total;
            }
            const uint8_t *gsrc = chunk_src(P, chunk);
            for (uint32_t i = tid; i < body; i += PACK_NT) gdst[hlen + i] = gsrc[i];
            if (crcHere && tid < 4) gdst[hlen + body + tid] = (uint8_t)((uint32_t)W->xxh >> (8 * tid));
        } else if (tid == 0) P.out_sizes[chunk] = -4;
        if (P.dbg_hdr && tid == 0) {
            uint32_t *d = P.dbg_hdr + (uint64_t)chunk * 4;
            d[0] = nseq; d[1] = nlit; d[2] = kind; d[3] = 0;
        }
    }
}

// ------------------------------------------------------------------------------------------------ K5
// XXH64 of every chunk (xxh64_quad, b2c_common.cuh): four lanes per chunk hold the four accumulators.
B2C_DEV void zstd_xxh_quad(const ZstdEncParams &P, uint32_t chunk, unsigned q /*0..3*/, unsigned quadBaseLane) {
    const bool live = chunk < P.nchunks;
    const uint8_t *src = chunk_src(P, live ? chunk : 0);
    uint32_t n = live ? chunk_size(P, chunk) : 0;
    const bool ok = n <= P.blockmax;
    if (!ok) n = 0;
    const uint64_t h = xxh64_quad(src, n, q, quadBaseLane);
    if (q == 0 && live && ok) P.work[chunk].xxh = h;
}

#ifndef B2C_EMU
extern "C" __global__ void __launch_bounds__(TABLES_NT, TABLES_MIN_CTAS) b2c_zstd_tables_kernel(ZstdEncParams P) {
    __shared__ TablesShared ts;
    if (threadIdx.x < 3) seq_build_predef(&ts.sw, (int)threadIdx.x);
    __syncthreads();
    zstd_tables_loop(&ts, P, blockIdx.x, gridDim.x);
}
// K3 + K5 in one launch: the three chain warps of a CTA walk the tANS chains of 32 chunks; when the launch has
// CHAIN_NT + CHAIN_XXH_NT threads, four more warps compute the XXH64 of the same 32 chunks (four lanes per chunk).  Both
// are latency-bound serial recurrences that need few registers, so they hide behind each other (as its own kernel XXH64
// cost 0.44 ms per GiB; a side stream beside the parse kernel did not overlap with it on the device).
extern "C" __global__ void __launch_bounds__(CHAIN_NT + CHAIN_XXH_NT) b2c_zstd_chains_kernel(ZstdEncParams P) {
    extern __shared__ __align__(1024) uint8_t smem[];
    if (threadIdx.x < CHAIN_NT) zstd_chains_block(reinterpret_cast<uint32_t *>(smem), P, blockIdx.x * 32);
    else {
        const unsigned t = threadIdx.x - CHAIN_NT;
        zstd_xxh_quad(P, blockIdx.x * 32 + (t >> 2), t & 3, (t & 31) & ~3u);
    }
}
extern "C" __global__ void __launch_bounds__(PACK_NT, PACK_MIN_CTAS) b2c_zstd_pack_kernel(ZstdEncParams P) {
    extern __shared__ __align__(1024) uint8_t smem[];
    zstd_pack_chunk<65536>(smem, P, blockIdx.x);
}
extern "C" __global__ void __launch_bounds__(PACK_NT, 1) b2c_zstd_pack128_kernel(ZstdEncParams P) {
    extern __shared__ __align__(1024) uint8_t smem[];
    zstd_pack_chunk<131072>(smem, P, blockIdx.x);
}
extern "C" __global__ void __launch_bounds__(128) b2c_zstd_xxh_kernel(ZstdEncParams P) {
    unsigned gt = blockIdx.x * blockDim.x + threadIdx.x;
    zstd_xxh_quad(P, gt >> 2, gt & 3, (threadIdx.x & 31) & ~3u);
}
#endif

}  // namespace b2c
