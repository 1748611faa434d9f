// compress_b200/csrc/b2c_lz4_cvt.cuh -- LZ4 / LZ4s block -> S2 / Snappy block conversion for sm_90a.
//
// What one LZ4Converter / LZ4sConverter ConvertBlock or ConvertBlockSnappy call does (s2/lz4convert.go:25-454,
// s2/lz4sconvert.go:30-467, the pure-Go code): the LZ4 token stream is rewritten tag by tag, without decompressing.  Two
// kernels, the shape of the staged S2 decoder:
//   walk  one LANE per block: the token walk decides the outcome exactly as the reference does (ErrCorrupt, and
//         ErrDstTooSmall from the size of every piece) and writes one 16-byte record per sequence that emits something
//   emit  one WARP per converted block: 32 records per step, output positions by a warp scan, every lane writes its tags,
//         literal runs are copied by their lane (short) or by the whole warp (long)
// Slot i receives uvarint(n) | body, so it is a complete S2 / Snappy block.  The decisions are the reference's for a dst
// with cap(dst) - len(dst) = slot capacity - 5, which leaves room for the header whatever n is.
#pragma once
#include "b2c_common.cuh"
#include "b2c_zstd_enc.cuh"

namespace b2c {

enum { LZC_LZ4 = 0, LZC_LZ4S = 1 };
enum { LZC_ERR_TOO_BIG = -3, LZC_ERR_DST = -4, LZC_ERR_CORRUPT = -5, LZC_ERR_ARG = -102 };

// Record of one sequence: literal run [lit, lit + ll) of the source block, then a match of ml bytes (0: none) at offset
// `off`; rep = the S2 output writes it as a repeat.
struct LzcRec { uint32_t lit, ll, ml, offRep; };
struct LzcHead { uint64_t n; uint32_t body, nrec; int32_t status; uint32_t pad; };

struct LzcParams {
    const uint8_t *src_base; uint64_t src_stride; const uint64_t *src_offsets; const uint32_t *src_sizes;
    uint8_t *dst_base; uint64_t dst_stride; const uint64_t *dst_offsets; const uint32_t *dst_caps; uint32_t dst_cap;
    int64_t *out_sizes, *decoded;
    uint32_t c0, nchunks;            // this pass: blocks c0 .. c0 + nchunks - 1
    int lz4s, snappy;
    LzcHead *heads;                  // [nchunks] of this pass
    LzcRec *recs;                    // block c's records at rec_base[c] - rec_base[c0], or (c - c0) * rec_per
    const uint64_t *rec_base; uint64_t rec_per;
};

// Record bound.  LZ4: every record but the last holds a match, so it took a token and two offset bytes; the last took a
// token and at least one literal: nrec <= (slen + 1) / 3.  LZ4s: a record without a match took a token and at least one
// literal (tokens with neither emit nothing), one with a match three bytes: nrec <= slen / 2.
B2C_DEV uint64_t lzc_rec_cap(uint64_t slen, int lz4s) { return (lz4s ? slen / 2 : slen / 3) + 1; }

// ---- emitters the S2 encoder's do not cover: literal headers of 4 and 5 bytes (runs > 64 KiB), copies and repeats of any
// length (emitRepeat16 splits a repeat above 2^24 - 1 + 2^16, s2/lz4convert.go:487-502) and the Snappy copy pieces of
// ConvertBlockSnappy (64-byte copy2 pieces, a remainder below 4 still copy2, s2/lz4convert.go:416-446)
constexpr uint64_t LZC_MAX_REP = (1u << 24) - 1 + (1u << 16);          // the longest repeat one 5-byte tag holds
B2C_DEV uint32_t lzc_lit_hdr_size(uint32_t ll) { return ll == 0 ? 0u : (ll <= 60 ? 1u : (ll <= 256 ? 2u : (ll <= 65536 ? 3u : (ll <= (1u << 24) ? 4u : 5u)))); }
B2C_DEV uint32_t lzc_put_lit_hdr(uint8_t *d, uint32_t ll) {
    if (ll <= 65536) return s2_put_lit_hdr(d, ll);
    const uint32_t n = ll - 1;
    d[1] = (uint8_t)n; d[2] = (uint8_t)(n >> 8); d[3] = (uint8_t)(n >> 16);
    if (n < (1u << 24)) { d[0] = 62 << 2; return 4; }
    d[0] = 63 << 2; d[4] = (uint8_t)(n >> 24);
    return 5;
}
B2C_DEV uint64_t lzc_repeat_size(uint32_t off, uint64_t len) {
    uint64_t sz = 0;
    while (len > LZC_MAX_REP + 4) { sz += 5; len -= LZC_MAX_REP; }
    return sz + s2_repeat_size(off, (uint32_t)len);
}
B2C_DEV uint32_t lzc_put_repeat(uint8_t *d, uint32_t off, uint64_t len) {
    uint32_t o = 0;
    while (len > LZC_MAX_REP + 4) { o += s2_put_repeat(d + o, off, (uint32_t)LZC_MAX_REP); len -= LZC_MAX_REP; }
    return o + s2_put_repeat(d + o, off, (uint32_t)len);
}
B2C_DEV uint64_t lzc_copy_size(uint32_t off, uint64_t len) {
    if (len > 64) return (off < 2048) ? 2 + lzc_repeat_size(off, len - 8) : 3 + lzc_repeat_size(off, len - 60);
    return s2_copy_size(off, (uint32_t)len);
}
B2C_DEV uint32_t lzc_put_copy(uint8_t *d, uint32_t off, uint64_t len) {
    if (len <= 64) return s2_put_copy(d, off, (uint32_t)len);
    uint32_t o;
    if (off < 2048) { d[1] = (uint8_t)off; d[0] = (uint8_t)((off >> 8) << 5 | (8 - 4) << 2 | 1); len -= 8; o = 2; }
    else { d[2] = (uint8_t)(off >> 8); d[1] = (uint8_t)off; d[0] = 59 << 2 | 2; len -= 60; o = 3; }
    return o + lzc_put_repeat(d + o, off, len);
}
B2C_DEV uint64_t lzc_snappy_size(uint32_t off, uint64_t len) {
    const uint64_t full = (len - 1) / 64, r = len - 64 * full;        // full 64-byte pieces, remainder 1 .. 64
    return 3 * full + ((r >= 12 || off >= 2048 || r < 4) ? 3u : 2u);
}
B2C_DEV uint32_t lzc_put_snappy(uint8_t *d, uint32_t off, uint64_t len) {
    uint32_t o = 0;
    while (len > 64) { d[o] = 63 << 2 | 2; d[o + 1] = (uint8_t)off; d[o + 2] = (uint8_t)(off >> 8); len -= 64; o += 3; }
    const uint32_t r = (uint32_t)len;
    if (r >= 12 || off >= 2048 || r < 4) { d[o] = (uint8_t)((r - 1) << 2 | 2); d[o + 1] = (uint8_t)off; d[o + 2] = (uint8_t)(off >> 8); return o + 3; }
    d[o + 1] = (uint8_t)off; d[o] = (uint8_t)((off >> 8) << 5 | (r - 4) << 2 | 1);
    return o + 2;
}
// A literal run copied by the whole warp: bytes up to the destination's 16-byte boundary, then 16-byte stores assembled
// from the aligned source words that hold them (read-only path), then the tail.
B2C_DEV void lzc_warp_copy(uint8_t *d, const uint8_t *s, uint32_t n, unsigned lane) {
    uint32_t head = (uint32_t)((16 - (reinterpret_cast<uintptr_t>(d) & 15)) & 15);
    if (head > n) head = n;
    if (lane < head) d[lane] = B2C_LDG(s + lane);
    const uint32_t body = (n - head) & ~15u;
    const uint32_t mis = (uint32_t)(reinterpret_cast<uintptr_t>(s + head) & 3), sh = mis * 8;
    const uint32_t *sw = reinterpret_cast<const uint32_t *>(s + head - mis);
    for (uint32_t i = lane * 16; i < body; i += 32 * 16) {
        const uint32_t *w = sw + (i >> 2);
        const uint32_t a0 = B2C_LDG(w), a1 = B2C_LDG(w + 1), a2 = B2C_LDG(w + 2), a3 = B2C_LDG(w + 3);
        const uint32_t a4 = mis ? B2C_LDG(w + 4) : 0u;                  // (holds source bytes only when mis != 0)
        uint4 v;
        v.x = __funnelshift_r(a0, a1, sh); v.y = __funnelshift_r(a1, a2, sh);
        v.z = __funnelshift_r(a2, a3, sh); v.w = __funnelshift_r(a3, a4, sh);
        *reinterpret_cast<uint4 *>(d + head + i) = v;
    }
    for (uint32_t i = head + body + lane; i < n; i += 32) d[i] = B2C_LDG(s + i);
}
B2C_DEV uint32_t lzc_uvarint_size(uint64_t v) { uint32_t n = 1; while (v >= 0x80) { v >>= 7; n++; } return n; }

B2C_DEV const uint8_t *lzc_src(const LzcParams &P, uint32_t c) { return P.src_base + (P.src_offsets ? P.src_offsets[c] : (uint64_t)c * P.src_stride); }
B2C_DEV LzcRec *lzc_recs(const LzcParams &P, uint32_t c) {
    return P.recs + (P.rec_base ? P.rec_base[c] - P.rec_base[P.c0] : (uint64_t)(c - P.c0) * P.rec_per);
}

// ---- walk: one lane per block
B2C_DEV void lzc_walk_lane(const LzcParams &P, uint32_t c) {
    const uint8_t *src = lzc_src(P, c);
    const uint32_t slen = P.src_sizes[c];
    const uint32_t cap = P.dst_caps ? P.dst_caps[c] : P.dst_cap;
    LzcHead *hd = P.heads + (c - P.c0);
    LzcRec *recs = lzc_recs(P, c);
    const uint64_t recCap = lzc_rec_cap(slen, P.lz4s);
    const bool s2 = !P.snappy;
    const uint32_t minMatch = P.lz4s ? 3 : 4;
    const int64_t dLimit = (int64_t)(cap > 5 ? cap - 5 : 0) - 10;
    // Bytes arrive as aligned words through the read-only path: byte i of the block is byte (i + mis) & 3 of word (i + mis) >> 2.
    const uint32_t mis = (uint32_t)(reinterpret_cast<uintptr_t>(src) & 3);
    const uint32_t *sw = reinterpret_cast<const uint32_t *>(src - mis);
    const uint32_t nsw = (uint32_t)(((uint64_t)slen + mis + 3) >> 2);
    auto word3 = [&](uint32_t pos) -> uint32_t {          // bytes pos .. pos + 2 (zero past the block's last word)
        const uint32_t wi = (uint32_t)(((uint64_t)pos + mis) >> 2), sh = ((pos + mis) & 3) * 8;
        const uint32_t w0 = B2C_LDG(sw + wi), w1 = wi + 1 < nsw ? B2C_LDG(sw + wi + 1) : 0u;
        return __funnelshift_r(w0, w1, sh);
    };
    int32_t status = 0;
    uint64_t unc = 0, d = 0, nrec = 0;
    uint32_t s = 0, lastOffset = 0;
    if (!P.rec_base && slen > P.src_stride) status = LZC_ERR_ARG;   // its records would not fit the room of a block
    while (slen > 0 && status == 0) {
        if (s >= slen) { status = LZC_ERR_CORRUPT; break; }
        const uint32_t token = word3(s) & 0xff;
        uint64_t ll = token >> 4, ml = minMatch + (token & 15);
        if (ll == 15) {
            uint32_t v;
            do {
                if (++s >= slen) { status = LZC_ERR_CORRUPT; break; }
                v = word3(s) & 0xff;
                ll += v;
            } while (v == 255);
            if (status) break;
        }
        if ((uint64_t)s + ll >= slen) { status = LZC_ERR_CORRUPT; break; }
        s++;
        const uint32_t lit = s;
        if (ll > 0) {
            if ((int64_t)(d + ll) > dLimit) { status = LZC_ERR_DST; break; }
            d += lzc_lit_hdr_size((uint32_t)ll) + ll;
            s += (uint32_t)ll;
            unc += ll;
        }
        const bool noMatch = ml == minMatch;
        if (noMatch && (P.lz4s || s == slen)) {                 // LZ4: the last token; LZ4s: a token without a match
            if (ll > 0) {
                if (nrec >= recCap) { status = LZC_ERR_CORRUPT; break; }   // (cannot happen: the record bound above)
                recs[nrec++] = LzcRec{lit, (uint32_t)ll, 0u, 0u};
            }
            if (s == slen) break;
            continue;
        }
        if (s + 2 >= slen) { status = LZC_ERR_CORRUPT; break; }
        const uint32_t ow = word3(s);
        const uint32_t off = ow & 0xffff;
        s += 2;
        if (off == 0 || off > unc) { status = LZC_ERR_CORRUPT; break; }
        if (ml == minMatch + 15) {
            uint32_t v = (ow >> 16) & 0xff;                     // (s < slen: checked above)
            s++;
            ml += v;
            while (v == 255) {
                if (s >= slen) { status = LZC_ERR_CORRUPT; break; }
                v = word3(s) & 0xff;
                s++;
                ml += v;
            }
            if (status) break;
            if (s >= slen) { status = LZC_ERR_CORRUPT; break; }
        }
        const bool rep = s2 && off == lastOffset;
        d += s2 ? (rep ? lzc_repeat_size(off, ml) : lzc_copy_size(off, ml)) : lzc_snappy_size(off, ml);
        if (s2) lastOffset = off;
        unc += ml;
        // One test for the reference's `d > dLimit` after the sequence, the Snappy form's `d >= dLimit` before every piece and
        // the inlined S2 emitters' room check: each of them fails exactly when the sequence ends past dLimit.
        if ((int64_t)d > dLimit) { status = LZC_ERR_DST; break; }
        if (nrec >= recCap) { status = LZC_ERR_CORRUPT; break; }       // (cannot happen: the record bound above)
        recs[nrec++] = LzcRec{lit, (uint32_t)ll, (uint32_t)(ml > 0xffffffffull ? 0xffffffffull : ml), off | (rep ? 1u << 16 : 0u)};
    }
    if (status == 0) {
        if (unc > 0xffffffffull) status = LZC_ERR_TOO_BIG;           // no S2 header can state it
        else if (lzc_uvarint_size(unc) + d > cap) status = LZC_ERR_DST;   // (only a slot below 5 bytes)
    }
    hd->n = unc; hd->body = (uint32_t)d; hd->nrec = (uint32_t)nrec; hd->status = status;
}

// ---- emit: one warp per block
B2C_DEV void lzc_emit_warp(const LzcParams &P, uint32_t c, unsigned lane) {
    const LzcHead hd = P.heads[c - P.c0];
    if (hd.status != 0) {
        if (lane == 0) { P.out_sizes[c] = hd.status; P.decoded[c] = hd.status == LZC_ERR_TOO_BIG ? (int64_t)hd.n : 0; }
        return;
    }
    const uint8_t *src = lzc_src(P, c);
    uint8_t *out = P.dst_base + (P.dst_offsets ? P.dst_offsets[c] : (uint64_t)c * P.dst_stride);
    const LzcRec *recs = lzc_recs(P, c);
    const uint32_t h = lzc_uvarint_size(hd.n);
    if (lane == 0) {
        uint64_t v = hd.n;
        for (uint32_t i = 0; i < h; i++, v >>= 7) out[i] = (uint8_t)(v | (i + 1 < h ? 0x80 : 0));
    }
    uint8_t *body = out + h;
    uint32_t d = 0;
    const bool s2 = !P.snappy;
    for (uint32_t base = 0; base < hd.nrec; base += 32) {
        const bool mine = base + lane < hd.nrec;
        const LzcRec r = mine ? recs[base + lane] : LzcRec{0, 0, 0, 0};
        const uint32_t off = r.offRep & 0xffff;
        const bool rep = (r.offRep >> 16) != 0;
        const uint32_t hb = lzc_lit_hdr_size(r.ll);
        const uint32_t cb = r.ml == 0 ? 0u : (uint32_t)(s2 ? (rep ? lzc_repeat_size(off, r.ml) : lzc_copy_size(off, r.ml)) : lzc_snappy_size(off, r.ml));
        const uint32_t sz = hb + r.ll + cb;
        const uint32_t incl = warp_scan_incl(sz);
        const uint32_t at = d + incl - sz;
        if (mine) {
            if (r.ll) lzc_put_lit_hdr(body + at, r.ll);
            if (r.ml) {
                uint8_t *t = body + at + hb + r.ll;
                if (s2) rep ? lzc_put_repeat(t, off, r.ml) : lzc_put_copy(t, off, r.ml);
                else lzc_put_snappy(t, off, r.ml);
            }
            if (r.ll <= 32) for (uint32_t i = 0; i < r.ll; i++) body[at + hb + i] = B2C_LDG(src + r.lit + i);
        }
        // longer runs: one at a time by the whole warp
        for (unsigned m = __ballot_sync(FULLMASK, r.ll > 32); m; m &= m - 1) {
            const int l = __popc((m & (0u - m)) - 1);                       // the lowest lane left
            const uint32_t n = __shfl_sync(FULLMASK, r.ll, l), from = __shfl_sync(FULLMASK, r.lit, l);
            const uint32_t to = __shfl_sync(FULLMASK, at + hb, l);
            lzc_warp_copy(body + to, src + from, n, lane);
        }
        d += __shfl_sync(FULLMASK, incl, 31);
    }
    __syncwarp();
    if (lane == 0) { P.out_sizes[c] = (int64_t)(h + hd.body); P.decoded[c] = (int64_t)hd.n; }
}

#ifndef B2C_EMU
constexpr int LZC_EMIT_WARPS = 4;
extern "C" __global__ void __launch_bounds__(32) b2c_lz4_cvt_walk_kernel(LzcParams P) {
    const uint32_t i = blockIdx.x * 32 + threadIdx.x;
    if (i < P.nchunks) lzc_walk_lane(P, P.c0 + i);
}
extern "C" __global__ void __launch_bounds__(LZC_EMIT_WARPS * 32) b2c_lz4_cvt_emit_kernel(LzcParams P) {
    const uint32_t i = blockIdx.x * LZC_EMIT_WARPS + (threadIdx.x >> 5);
    if (i < P.nchunks) lzc_emit_warp(P, P.c0 + i, threadIdx.x & 31);
}
#endif

}  // namespace b2c
