/*
 * oracle/orc_lz4.c -- LZ4 / LZ4s -> S2 / Snappy block converter oracle.  TEST INFRASTRUCTURE ONLY (see orc_common.h).
 *
 * Restates the reference's pure-Go code (the amd64 assembler twins cvtLZ4*Asm are not restated):
 *   LZ4Converter.ConvertBlock / ConvertBlockSnappy     s2/lz4convert.go:25-275, 281-454
 *   LZ4sConverter.ConvertBlock / ConvertBlockSnappy    s2/lz4sconvert.go:30-284, 290-467
 *   emitRepeat16 / emitCopy16 / emitLiteralGo          s2/lz4convert.go:456-585
 * and, so that LZ4 and LZ4s inputs can be produced and checked on every machine,
 *   lz4ref CompressBlock / CompressBlockLZ4s / UncompressBlock   internal/lz4ref/block.go:82-515, 517-655
 *
 * One deliberate deviation: ConvertBlock's inlined copy / repeat emitters (lz4convert.go:158-267) only check that more
 * than 5 bytes are left in dst.  A copy or repeat whose tag bytes need more room than is left (reachable after a literal
 * run with a 3- to 5-byte header that ends just below the limit, or with a repeat longer than 2^24 that is split) indexes
 * past dst, which panics in Go.  Here, as in the device kernels, that case is ErrDstTooSmall.
 */
#include "orc_common.h"
#include <stdlib.h>

#define TAG_LITERAL 0x00
#define TAG_COPY1 0x01
#define TAG_COPY2 0x02

/* A bounded output: bytes written at or past `cap` are dropped and flag an overflow (where Go would panic). */
typedef struct { uint8_t *p; int64_t cap; int ovf; } obuf;
static void put(obuf *o, int64_t i, uint8_t v) {
    if (i >= 0 && i < o->cap) o->p[i] = v;
    else o->ovf = 1;
}

/* emitRepeat16 (lz4convert.go:456-503) at o[at]; returns the bytes written */
static int64_t emit_repeat16(obuf *o, int64_t at, uint16_t offset, int64_t length) {
    length -= 4;
    if (length <= 4) { put(o, at, (uint8_t)(length << 2 | TAG_COPY1)); put(o, at + 1, 0); return 2; }
    if (length < 8 && offset < 2048) {
        put(o, at + 1, (uint8_t)offset);
        put(o, at, (uint8_t)((offset >> 8) << 5 | length << 2 | TAG_COPY1));
        return 2;
    }
    if (length < (1 << 8) + 4) {
        length -= 4;
        put(o, at + 2, (uint8_t)length); put(o, at + 1, 0); put(o, at, 5 << 2 | TAG_COPY1);
        return 3;
    }
    if (length < (1 << 16) + (1 << 8)) {
        length -= 1 << 8;
        put(o, at + 3, (uint8_t)(length >> 8)); put(o, at + 2, (uint8_t)length); put(o, at + 1, 0); put(o, at, 6 << 2 | TAG_COPY1);
        return 4;
    }
    const int64_t maxRepeat = (1 << 24) - 1;
    length -= 1 << 16;
    int64_t left = 0;
    if (length > maxRepeat) { left = length - maxRepeat + 4; length = maxRepeat - 4; }
    put(o, at + 4, (uint8_t)(length >> 16)); put(o, at + 3, (uint8_t)(length >> 8)); put(o, at + 2, (uint8_t)length);
    put(o, at + 1, 0); put(o, at, 7 << 2 | TAG_COPY1);
    if (left > 0) return 5 + emit_repeat16(o, at + 5, offset, left);
    return 5;
}

/* emitCopy16 (lz4convert.go:505-544) */
static int64_t emit_copy16(obuf *o, int64_t at, uint16_t offset, int64_t length) {
    if (length > 64) {
        int64_t off = 3;
        if (offset < 2048) {
            put(o, at + 1, (uint8_t)offset);
            put(o, at, (uint8_t)((offset >> 8) << 5 | (8 - 4) << 2 | TAG_COPY1));
            length -= 8;
            off = 2;
        } else {
            put(o, at + 2, (uint8_t)(offset >> 8)); put(o, at + 1, (uint8_t)offset); put(o, at, 59 << 2 | TAG_COPY2);
            length -= 60;
        }
        return off + emit_repeat16(o, at + off, offset, length);
    }
    if (length >= 12 || offset >= 2048) {
        put(o, at + 2, (uint8_t)(offset >> 8)); put(o, at + 1, (uint8_t)offset); put(o, at, (uint8_t)((length - 1) << 2 | TAG_COPY2));
        return 3;
    }
    put(o, at + 1, (uint8_t)offset);
    put(o, at, (uint8_t)((offset >> 8) << 5 | (length - 4) << 2 | TAG_COPY1));
    return 2;
}

/* emitLiteralGo (lz4convert.go:552-585) */
static int64_t emit_literal(obuf *o, int64_t at, const uint8_t *lit, int64_t len) {
    if (len == 0) return 0;
    int64_t i;
    const uint64_t n = (uint64_t)len - 1;
    if (n < 60) { put(o, at, (uint8_t)(n << 2 | TAG_LITERAL)); i = 1; }
    else if (n < (1u << 8)) { put(o, at + 1, (uint8_t)n); put(o, at, 60 << 2 | TAG_LITERAL); i = 2; }
    else if (n < (1u << 16)) { put(o, at + 2, (uint8_t)(n >> 8)); put(o, at + 1, (uint8_t)n); put(o, at, 61 << 2 | TAG_LITERAL); i = 3; }
    else if (n < (1u << 24)) {
        put(o, at + 3, (uint8_t)(n >> 16)); put(o, at + 2, (uint8_t)(n >> 8)); put(o, at + 1, (uint8_t)n); put(o, at, 62 << 2 | TAG_LITERAL);
        i = 4;
    } else {
        put(o, at + 4, (uint8_t)(n >> 24)); put(o, at + 3, (uint8_t)(n >> 16)); put(o, at + 2, (uint8_t)(n >> 8)); put(o, at + 1, (uint8_t)n);
        put(o, at, 63 << 2 | TAG_LITERAL);
        i = 5;
    }
    if (at + i + len <= o->cap) memcpy(o->p + at + i, lit, (size_t)len);
    else o->ovf = 1;
    return i + len;
}

/*
 * One conversion.  dst[0, dlen) is the existing content of the Go slice, dcap its capacity; src the LZ4 (lz4s = 0) or LZ4s
 * (lz4s = 1) block.  snappy = 0: ConvertBlock, 1: ConvertBlockSnappy.  Returns the new length of dst, or ORC_ERR_CORRUPT
 * (ErrCorrupt) / ORC_ERR_DST_SMALL (ErrDstTooSmall); *n_out = the decoded size on success.
 */
ORC_API int64_t orc_lz4_convert(int lz4s, int snappy, uint8_t *dst, int64_t dlen, int64_t dcap, const uint8_t *src, int64_t slen,
                                int64_t *n_out) {
    *n_out = 0;
    if (slen == 0) return dlen;
    const int64_t minMatch = lz4s ? 3 : 4;
    obuf o = {dst, dcap, 0};
    int64_t s = 0, d = dlen;
    const int64_t dLimit = dcap - 10;
    uint16_t lastOffset = 0;
    int64_t uncompressed = 0;
    for (;;) {
        if (s >= slen) return ORC_ERR_CORRUPT;
        const uint8_t token = src[s];
        int64_t ll = token >> 4;
        int64_t ml = minMatch + (token & 0xf);
        if (token >= 0xf0) {
            for (;;) {
                s++;
                if (s >= slen) return ORC_ERR_CORRUPT;
                const uint8_t val = src[s];
                ll += val;
                if (val != 255) break;
            }
        }
        if (s + ll >= slen) return ORC_ERR_CORRUPT;
        s++;
        if (ll > 0) {
            if (d + ll > dLimit) return ORC_ERR_DST_SMALL;
            d += emit_literal(&o, d, src + s, ll);
            s += ll;
            uncompressed += ll;
        }
        if (lz4s) {                                  /* lz4sconvert.go:115-122: ml == minMatch is "no match" */
            if (ml == minMatch) {
                if (s == slen) break;
                continue;
            }
        } else if (s == slen && ml == minMatch) break;   /* lz4convert.go:110-113 */
        if (s >= slen - 2) return ORC_ERR_CORRUPT;
        const uint16_t offset = (uint16_t)(src[s] | src[s + 1] << 8);
        s += 2;
        if (offset == 0) return ORC_ERR_CORRUPT;
        if ((int64_t)offset > uncompressed) return ORC_ERR_CORRUPT;
        if (ml == minMatch + 15) {
            for (;;) {
                if (s >= slen) return ORC_ERR_CORRUPT;
                const uint8_t val = src[s];
                s++;
                ml += val;
                if (val != 255) {
                    if (s >= slen) return ORC_ERR_CORRUPT;
                    break;
                }
            }
        }
        if (snappy) {                                /* lz4convert.go:416-446: 64-byte copy2 pieces, no repeats */
            int64_t length = ml;
            while (length > 0) {
                if (d >= dLimit) return ORC_ERR_DST_SMALL;
                if (length > 64) {
                    put(&o, d + 2, (uint8_t)(offset >> 8)); put(&o, d + 1, (uint8_t)offset); put(&o, d, 63 << 2 | TAG_COPY2);
                    length -= 64;
                    d += 3;
                    continue;
                }
                if (length >= 12 || offset >= 2048 || length < 4) {
                    put(&o, d + 2, (uint8_t)(offset >> 8)); put(&o, d + 1, (uint8_t)offset);
                    put(&o, d, (uint8_t)((length - 1) << 2 | TAG_COPY2));
                    d += 3;
                    break;
                }
                put(&o, d + 1, (uint8_t)offset);
                put(&o, d, (uint8_t)((offset >> 8) << 5 | (length - 4) << 2 | TAG_COPY1));
                d += 2;
                break;
            }
        } else if (dcap - d > 5) {                   /* the inlined loops' `for len(dst) > 5` (lz4convert.go:167, 229) */
            if (offset == lastOffset) d += emit_repeat16(&o, d, offset, ml);
            else d += emit_copy16(&o, d, offset, ml);
            if (o.ovf) return ORC_ERR_DST_SMALL;     /* Go: index out of range (see the header comment) */
        }
        if (!snappy && offset != lastOffset) lastOffset = offset;
        uncompressed += ml;
        if (d > dLimit) return ORC_ERR_DST_SMALL;
    }
    if (o.ovf) return ORC_ERR_DST_SMALL;             /* (cannot happen: every literal run is checked against dLimit) */
    *n_out = uncompressed;
    return d;
}

/* ---- lz4ref (internal/lz4ref/block.go) -------------------------------------------------------------- */
#define LZ4_MIN_MATCH 4
#define LZ4_WIN_SIZE (1 << 16)
#define LZ4_WIN_MASK (LZ4_WIN_SIZE - 1)
#define LZ4_HASH_LOG 16
#define LZ4_HT_SIZE (1 << LZ4_HASH_LOG)
#define LZ4_MF_LIMIT (10 + LZ4_MIN_MATCH)

static uint64_t le64(const uint8_t *p) { uint64_t v; memcpy(&v, p, 8); return v; }
static uint32_t le32(const uint8_t *p) { uint32_t v; memcpy(&v, p, 4); return v; }
static uint32_t block_hash(uint64_t x) {            /* block.go:28-32 */
    const uint64_t prime6bytes = 227718039650203ull;
    x &= ((uint64_t)1 << 40) - 1;
    return (uint32_t)((x * prime6bytes) >> (64 - LZ4_HASH_LOG));
}
typedef struct { uint16_t table[LZ4_HT_SIZE]; uint32_t inUse[LZ4_HT_SIZE / 32]; } lz4c;
static int64_t lz4c_get(const lz4c *c, uint32_t h, int64_t si) {   /* block.go:58-70 */
    h &= LZ4_HT_SIZE - 1;
    int64_t i = 0;
    if (c->inUse[h / 32] & (1u << (h % 32))) i = c->table[h];
    i += si & ~(int64_t)LZ4_WIN_MASK;
    if (i >= si) i -= LZ4_WIN_SIZE;
    return i;
}
static void lz4c_put(lz4c *c, uint32_t h, int64_t si) {
    h &= LZ4_HT_SIZE - 1;
    c->table[h] = (uint16_t)si;
    c->inUse[h / 32] |= 1u << (h % 32);
}
static int tz64(uint64_t x) { return __builtin_ctzll(x); }

ORC_API int64_t orc_lz4_compress_bound(int64_t n) { return n + n / 255 + 16; }   /* CompressBlockBound, block.go:34-36 */

/*
 * Compressor.CompressBlock (lz4s = 0, block.go:96-298) / CompressBlockLZ4s (lz4s = 1, :300-515).  Returns the block's
 * size, 0 for "incompressible" (dst smaller than CompressBlockBound and nothing found), or -1 for
 * ErrInvalidSourceShortBuffer.  The LZ4s form cuts 32 literals off every longer literal run into a token of its own with
 * no match (addExtraLits, :306), so that its output holds the zero-match tokens real LZ4s producers write.
 */
ORC_API int64_t orc_lz4_compress_block(int lz4s, const uint8_t *src, int64_t slen, uint8_t *dst, int64_t dlen) {
    lz4c *c = (lz4c *)calloc(1, sizeof(lz4c));
    if (!c) return -1;
    const int64_t minMatch = lz4s ? 3 : 4, addExtraLits = 32;
    const int isNotCompressible = dlen < orc_lz4_compress_bound(slen);
    const int adaptSkipLog = 7;
    int64_t si = 0, di = 0, anchor = 0, r = 0;
    const int64_t sn = slen - LZ4_MF_LIMIT;
#define SHORT() do { r = -1; goto out; } while (0)
    if (sn <= 0) goto lastLiterals;
    while (si < sn) {
        const uint64_t match = le64(src + si);
        uint32_t h = block_hash(match), h2 = block_hash(match >> 8);
        const int64_t ref = lz4c_get(c, h, si), ref2 = lz4c_get(c, h2, si + 1);
        lz4c_put(c, h, si);
        lz4c_put(c, h2, si + 1);
        int64_t offset = si - ref;
        if (offset <= 0 || offset >= LZ4_WIN_SIZE || (uint32_t)match != le32(src + ref)) {
            h = block_hash(match >> 16);
            const int64_t ref3 = lz4c_get(c, h, si + 2);
            si += 1;
            offset = si - ref2;
            if (offset <= 0 || offset >= LZ4_WIN_SIZE || (uint32_t)(match >> 8) != le32(src + ref2)) {
                si += 1;
                offset = si - ref3;
                lz4c_put(c, h, si);
                if (offset <= 0 || offset >= LZ4_WIN_SIZE || (uint32_t)(match >> 16) != le32(src + ref3)) {
                    si += 2 + ((si - anchor) >> adaptSkipLog);
                    continue;
                }
            }
        }
        int64_t lLen = si - anchor, mLen = 4;
        int64_t tOff = si - offset - 1;
        while (lLen > 0 && tOff >= 0 && src[si - 1] == src[tOff]) { si--; tOff--; lLen--; mLen++; }
        { const int64_t base = si + minMatch; si = si + mLen; mLen = base; }
        while (si + 8 <= sn) {
            const uint64_t x = le64(src + si) ^ le64(src + si - offset);
            if (x == 0) si += 8;
            else { si += tz64(x) >> 3; break; }
        }
        if (lz4s && lLen > addExtraLits) {           /* block.go:397-408 */
            if (di + 2 + addExtraLits > dlen) SHORT();
            dst[di] = 0xf0;
            dst[di + 1] = (uint8_t)(addExtraLits - 15);
            di += 2;
            memcpy(dst + di, src + anchor, (size_t)addExtraLits);
            di += addExtraLits;
            lLen -= addExtraLits;
            anchor += addExtraLits;
        }
        mLen = si - mLen;
        if (di >= dlen) SHORT();
        dst[di] = mLen < 0xF ? (uint8_t)mLen : 0xF;
        if (lLen < 0xF) dst[di] |= (uint8_t)(lLen << 4);
        else {
            dst[di] |= 0xF0;
            di++;
            int64_t l = lLen - 0xF;
            for (; l >= 0xFF && di < dlen; l -= 0xFF) dst[di++] = 0xFF;
            if (di >= dlen) SHORT();
            dst[di] = (uint8_t)l;
        }
        di++;
        if (di + lLen > dlen) SHORT();
        memcpy(dst + di, src + anchor, (size_t)lLen);
        di += lLen + 2;
        anchor = si;
        if (di > dlen) SHORT();
        dst[di - 2] = (uint8_t)offset; dst[di - 1] = (uint8_t)(offset >> 8);
        if (mLen >= 0xF) {
            for (mLen -= 0xF; mLen >= 0xFF && di < dlen; mLen -= 0xFF) dst[di++] = 0xFF;
            if (di >= dlen) SHORT();
            dst[di++] = (uint8_t)mLen;
        }
        if (si >= sn) break;
        h = block_hash(le64(src + si - 2));
        lz4c_put(c, h, si - 2);
    }
lastLiterals:
    if (isNotCompressible && anchor == 0) { r = 0; goto out; }
    if (di >= dlen) SHORT();
    {
        int64_t lLen = slen - anchor;
        if (lLen < 0xF) dst[di] = (uint8_t)(lLen << 4);
        else {
            dst[di] = 0xF0;
            di++;
            for (lLen -= 0xF; lLen >= 0xFF && di < dlen; lLen -= 0xFF) dst[di++] = 0xFF;
            if (di >= dlen) SHORT();
            dst[di] = (uint8_t)lLen;
        }
        di++;
    }
    if (isNotCompressible && di >= anchor) { r = 0; goto out; }
    if (di + slen - anchor > dlen) SHORT();
    memcpy(dst + di, src + anchor, (size_t)(slen - anchor));
    di += slen - anchor;
    r = di;
#undef SHORT
out:
    free(c);
    return r;
}

/*
 * UncompressBlock (block.go:517-655): the decoded size, or -2 (hasError) for a malformed block or one that does not fit
 * dst[0, dcap).  The reference's 16- and 18-byte shortcut copies give the same result as the general path restated here: a
 * shortcut that runs past dst only ever ends in the error a later bounds check reports.
 */
ORC_API int64_t orc_lz4_uncompress_block(uint8_t *dst, int64_t dcap, const uint8_t *src, int64_t slen) {
    const int64_t hasError = -2;
    if (slen == 0) return hasError;
    uint64_t si = 0, di = 0;
    const uint64_t n = (uint64_t)slen, cap = (uint64_t)dcap;
    for (;;) {
        if (si >= n) return hasError;
        const uint64_t b = src[si++];
        uint64_t lLen = b >> 4;
        if (lLen > 0) {
            if (lLen == 0xF) {
                for (;;) {
                    if (si >= n) return hasError;
                    const uint64_t x = src[si];
                    lLen += x;
                    si++;
                    if (x != 0xFF) break;
                }
            }
            if (si + lLen > n || di + lLen > cap) return hasError;
            memcpy(dst + di, src + si, (size_t)lLen);
            si += lLen;
            di += lLen;
        }
        uint64_t mLen = b & 0xF;
        if (si == n && mLen == 0) break;
        if (n < 2 || si >= n - 2) return hasError;
        const uint64_t offset = (uint64_t)src[si] | (uint64_t)src[si + 1] << 8;
        if (offset == 0) return hasError;
        si += 2;
        mLen += LZ4_MIN_MATCH;
        if (mLen == LZ4_MIN_MATCH + 0xF) {
            for (;;) {
                if (si >= n) return hasError;
                const uint64_t x = src[si];
                mLen += x;
                si++;
                if (x != 0xFF) break;
            }
        }
        if (di < offset) return hasError;
        if (di + mLen > cap) return hasError;
        for (uint64_t k = 0; k < mLen; k++) dst[di + k] = dst[di - offset + k];
        di += mLen;
    }
    return (int64_t)di;
}
