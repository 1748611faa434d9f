/*
 * oracle/orc_s2best.c -- the S2 "best" block encoders.  TEST INFRASTRUCTURE ONLY (see orc_common.h).
 *
 * Built as its own library (oracle/s2best.mk) around the unchanged S2 oracle, which it compiles in (emitters, decoder and
 * the Encode / EncodeBetter / EncodeSnappy wrappers keep their behaviour bit for bit).  It restates, without a dictionary:
 *   encodeBlockBest, encodeBlockBestSnappy           s2/encode_best.go:22-447, 457-716
 *   emitCopySize, emitCopyNoRepeatSize, emitRepeatSize   s2/encode_best.go:718-800
 *   EncodeBest / EncodeSnappyBest wrappers           s2/encode.go:161-188, 292-320
 * and exposes them as modes 3 (EncodeBest) and 4 (EncodeSnappyBest) of orc_s2x_encode / orc_s2x_encode_block, which
 * pass modes 0-2 to orc_s2_encode / orc_s2_encode_block.
 */
#include "orc_s2.c"

#define BEST_LBITS 19           /* bestLongTableBits,  s2/hashtable_pool.go:16-20 */
#define BEST_SBITS 16           /* bestShortTableBits */
#define BEST_MARGIN (8 + 2)     /* inputMargin */
#define BEST_MAXSKIP 64

static inline uint32_t hash8(uint64_t u, unsigned h) { return (uint32_t)((u * 0xcf1bbcdcb7a56463ull) >> (64 - h)); }

/* ---- size helpers (s2/encode_best.go:718-800) ------------------------------------------------------ */
ORC_API int64_t orc_s2_emit_repeat_size(int64_t offset, int64_t length) {
    if (length <= 4 + 4 || (length < 8 + 4 && offset < 2048)) return 2;
    if (length < (1 << 8) + 4 + 4) return 3;
    if (length < (1 << 16) + (1 << 8) + 4) return 4;
    const int64_t maxRepeat = (1 << 24) - 1;
    length -= (1 << 16) - 4;
    int64_t left = 0;
    if (length > maxRepeat) left = length - maxRepeat + 4;
    if (left > 0) return 5 + orc_s2_emit_repeat_size(offset, left);
    return 5;
}

ORC_API int64_t orc_s2_emit_copy_size(int64_t offset, int64_t length) {
    if (offset >= 65536) {
        int64_t i = 0;
        if (length > 64) {
            length -= 64;
            if (length >= 4) return 5 + orc_s2_emit_repeat_size(offset, length);
            i = 5;
        }
        if (length == 0) return i;
        return i + 5;
    }
    if (length > 64) {
        if (offset < 2048) return 2 + orc_s2_emit_repeat_size(offset, length - 8);
        return 3 + orc_s2_emit_repeat_size(offset, length - 60);
    }
    if (length >= 12 || offset >= 2048) return 3;
    return 2;
}

ORC_API int64_t orc_s2_emit_copy_norepeat_size(int64_t offset, int64_t length) {
    if (offset >= 65536) return 5 + 5 * (length / 64);
    if (length > 64) return 3 + 3 * (length / 60);
    if (length >= 12 || offset >= 2048) return 3;
    return 2;
}

/* First length in [lmin, lmax] where a size helper differs from what its emitter writes, or -1.
 * which: 0 emitCopySize / emitCopy, 1 emitRepeatSize / emitRepeat, 2 emitCopyNoRepeatSize / emitCopyNoRepeat. */
ORC_API int64_t orc_s2_size_helper_mismatch(int which, int64_t offset, int64_t lmin, int64_t lmax) {
    uint8_t buf[64];
    for (int64_t l = lmin; l <= lmax; l++) {
        int64_t want, got;
        if (which == 0) { want = orc_s2_emit_copy(buf, offset, l); got = orc_s2_emit_copy_size(offset, l); }
        else if (which == 1) { want = orc_s2_emit_repeat(buf, offset, l); got = orc_s2_emit_repeat_size(offset, l); }
        else { want = orc_s2_emit_copy_norepeat(buf, offset, l); got = orc_s2_emit_copy_norepeat_size(offset, l); }
        if (want != got) return l;
    }
    return -1;
}

/* ---- encodeBlockBest / encodeBlockBestSnappy ------------------------------------------------------ */
typedef struct { int64_t offset, s, length, score; int rep; } best_match;

typedef struct {
    const uint8_t *src;
    int64_t n, sLimit, nextEmit;
    int snappy;
    best_match best;     /* the search's current best: matchAt skips a candidate with its offset */
} best_state;

static int64_t best_score(const best_state *B, const best_match *m) {
    int64_t score = m->length - m->s;
    if (B->nextEmit == m->s) score++;        /* no literal has to be emitted */
    const int64_t offset = m->s - m->offset;
    if (B->snappy) return score - orc_s2_emit_copy_norepeat_size(offset, m->length);
    if (m->rep) return score - orc_s2_emit_repeat_size(offset, m->length);
    return score - orc_s2_emit_copy_size(offset, m->length);
}

static best_match match_at(const best_state *B, int64_t offset, int64_t s, uint32_t first, int rep) {
    const uint8_t *src = B->src;
    best_match m = {offset, s, 0, 0, rep};
    if (B->best.length != 0 && B->best.s - B->best.offset == s - offset) return m;   /* same offset: not retested */
    if (orc_ld32(src + offset) != first) return m;
    m.length = 4 + offset;
    s += 4;
    if (B->snappy) {          /* encode_best.go:541-547: 8 bytes at a time up to sLimit */
        while (s <= B->sLimit) {
            uint64_t diff = orc_ld64(src + s) ^ orc_ld64(src + m.length);
            if (diff != 0) { m.length += __builtin_ctzll(diff) >> 3; break; }
            s += 8; m.length += 8;
        }
    } else {                  /* encode_best.go:134-148: to the end of the block */
        while (s < B->n) {
            if (B->n - s < 8) {
                if (src[s] == src[m.length]) { m.length++; s++; continue; }
                break;
            }
            uint64_t diff = orc_ld64(src + s) ^ orc_ld64(src + m.length);
            if (diff != 0) { m.length += __builtin_ctzll(diff) >> 3; break; }
            s += 8; m.length += 8;
        }
    }
    m.length -= offset;
    m.score = best_score(B, &m);
    if (m.score <= -m.s) m.length = 0;       /* no saving */
    return m;
}

static best_match best_of(best_match a, best_match b) {
    if (b.length == 0) return a;
    if (a.length == 0) return b;
    return (a.score + b.s >= b.score + a.s) ? a : b;
}

#define CUR(x) ((int64_t)((x) & 0xffffffffu))
#define PREV(x) ((int64_t)((x) >> 32))

static int64_t encode_block_best(uint8_t *dst, const uint8_t *src, int64_t n, int snappy) {
    best_state B;
    memset(&B, 0, sizeof(B));
    B.src = src; B.n = n; B.sLimit = n - BEST_MARGIN; B.snappy = snappy;
    if (n < MIN_NON_LITERAL) return 0;
    uint64_t *lTable = (uint64_t *)calloc((size_t)1 << BEST_LBITS, sizeof(uint64_t));
    uint64_t *sTable = (uint64_t *)calloc((size_t)1 << BEST_SBITS, sizeof(uint64_t));
    if (!lTable || !sTable) { free(lTable); free(sTable); return ORC_ERR_INTERNAL; }
#define RET(v) do { free(lTable); free(sTable); return (v); } while (0)
    const int64_t sLimit = B.sLimit, dstLimit = n - 5;
    int64_t s = 1, d = 0, repeat = 1;
    uint64_t cv = orc_ld64(src + s);
    for (;;) {
        memset(&B.best, 0, sizeof(B.best));      /* `var best match`: every search starts without a match */
        for (;;) {
            int64_t nextS = ((s - B.nextEmit) >> 8) + 1;
            nextS = nextS > BEST_MAXSKIP ? s + BEST_MAXSKIP : nextS + s;
            if (nextS > sLimit) goto emitRemainder;
            const uint32_t hashL = hash8(cv, BEST_LBITS), hashS = hash4(cv, BEST_SBITS);
            const uint64_t candidateL = lTable[hashL], candidateS = sTable[hashS];
            best_match m0, m1;
            if (s > 0) {
                m0 = match_at(&B, CUR(candidateL), s, (uint32_t)cv, 0);
                m1 = match_at(&B, PREV(candidateL), s, (uint32_t)cv, 0);
                B.best = best_of(m0, m1);
                B.best = best_of(B.best, match_at(&B, CUR(candidateS), s, (uint32_t)cv, 0));
                B.best = best_of(B.best, match_at(&B, PREV(candidateS), s, (uint32_t)cv, 0));
            }
            if (repeat > 0) B.best = best_of(B.best, match_at(&B, s - repeat + 1, s + 1, (uint32_t)(cv >> 8), !snappy));
            if (B.best.length > 0) {
                /* s+1 */
                uint64_t nextShort = sTable[hash4(cv >> 8, BEST_SBITS)];
                int64_t s1 = s + 1;
                uint64_t cv1 = orc_ld64(src + s1);
                uint64_t nextLong = lTable[hash8(cv1, BEST_LBITS)];
                B.best = best_of(B.best, match_at(&B, CUR(nextShort), s1, (uint32_t)cv1, 0));
                B.best = best_of(B.best, match_at(&B, PREV(nextShort), s1, (uint32_t)cv1, 0));
                B.best = best_of(B.best, match_at(&B, CUR(nextLong), s1, (uint32_t)cv1, 0));
                B.best = best_of(B.best, match_at(&B, PREV(nextLong), s1, (uint32_t)cv1, 0));
                if (snappy)   /* "repeat at +2" of the Snappy form: the repeat candidate at s1 + 1 */
                    B.best = best_of(B.best, match_at(&B, s1 - repeat + 1, s1 + 1, (uint32_t)(cv1 >> 8), 0));
                /* s+2 */
                nextShort = sTable[hash4(cv1 >> 8, BEST_SBITS)];
                s1++;
                cv1 = orc_ld64(src + s1);
                nextLong = lTable[hash8(cv1, BEST_LBITS)];
                if (!snappy && repeat > 0) B.best = best_of(B.best, match_at(&B, s1 - repeat, s1, (uint32_t)cv1, 1));
                B.best = best_of(B.best, match_at(&B, CUR(nextShort), s1, (uint32_t)cv1, 0));
                B.best = best_of(B.best, match_at(&B, PREV(nextShort), s1, (uint32_t)cv1, 0));
                B.best = best_of(B.best, match_at(&B, CUR(nextLong), s1, (uint32_t)cv1, 0));
                B.best = best_of(B.best, match_at(&B, PREV(nextLong), s1, (uint32_t)cv1, 0));
                /* match end: long-table candidates at the best match's end, shifted back by its length.  S2 allows the
                 * first two bytes to mismatch (skipBeginning 2, skipEnd 1); Snappy probes the exact end. */
                const int64_t skipB = snappy ? 0 : 2, skipE = snappy ? 0 : 1;
                const int64_t sAt = B.best.s + B.best.length - skipE;
                if (sAt < sLimit) {
                    const int64_t sBack = B.best.s + skipB - skipE, backL = B.best.length - skipB;
                    const uint64_t cvb = orc_ld64(src + sBack);
                    const uint64_t next = lTable[hash8(orc_ld64(src + sAt), BEST_LBITS)];
                    int64_t checkAt = CUR(next) - backL;
                    if (checkAt > 0) B.best = best_of(B.best, match_at(&B, checkAt, sBack, (uint32_t)cvb, 0));
                    checkAt = PREV(next) - backL;
                    if (checkAt > 0) B.best = best_of(B.best, match_at(&B, checkAt, sBack, (uint32_t)cvb, 0));
                }
            }
            lTable[hashL] = (uint64_t)s | candidateL << 32;
            sTable[hashS] = (uint64_t)s | candidateS << 32;
            if (B.best.length > 0) break;
            cv = orc_ld64(src + nextS);
            s = nextS;
        }
        /* extend backwards (not for repeats) */
        s = B.best.s;
        if (!B.best.rep)
            while (B.best.offset > 0 && s > B.nextEmit && src[B.best.offset - 1] == src[s - 1]) { B.best.offset--; B.best.length++; s--; }
        if (d + (s - B.nextEmit) > dstLimit) RET(0);
        const int64_t base = s, offset = s - B.best.offset;
        s += B.best.length;
        if (offset > 65535 && s - base <= 5 && !B.best.rep) {
            s = B.best.s + 1;
            if (s >= sLimit) goto emitRemainder;
            cv = orc_ld64(src + s);
            continue;
        }
        d += orc_s2_emit_literal(dst + d, src + B.nextEmit, (size_t)(base - B.nextEmit));
        if (snappy) d += orc_s2_emit_copy_norepeat(dst + d, offset, B.best.length);
        else if (B.best.rep && B.nextEmit > 0) d += orc_s2_emit_repeat(dst + d, offset, B.best.length);
        else d += orc_s2_emit_copy(dst + d, offset, B.best.length);
        repeat = offset;
        B.nextEmit = s;
        if (s >= sLimit) goto emitRemainder;
        if (d > dstLimit) RET(0);
        for (int64_t i = B.best.s + 1; i < s; i++) {
            const uint64_t cv0 = orc_ld64(src + i);
            const uint32_t long0 = hash8(cv0, BEST_LBITS), short0 = hash4(cv0, BEST_SBITS);
            lTable[long0] = (uint64_t)i | lTable[long0] << 32;
            sTable[short0] = (uint64_t)i | sTable[short0] << 32;
        }
        cv = orc_ld64(src + s);
    }
emitRemainder:
    if (B.nextEmit < n) {
        if (d + n - B.nextEmit > dstLimit) RET(0);
        d += orc_s2_emit_literal(dst + d, src + B.nextEmit, (size_t)(n - B.nextEmit));
    }
    RET(d);
#undef RET
}
#undef CUR
#undef PREV

/* mode 0-2 as orc_s2_encode_block; 3 encodeBlockBest, 4 encodeBlockBestSnappy.  The block body, 0 = not compressible. */
ORC_API int64_t orc_s2x_encode_block(uint8_t *dst, const uint8_t *src, int64_t n, int mode) {
    if (mode == 3 || mode == 4) return encode_block_best(dst, src, n, mode == 4);
    return orc_s2_encode_block(dst, src, n, mode);
}

/* Encode / EncodeBetter / EncodeSnappy (modes 0-2) and EncodeBest / EncodeSnappyBest (modes 3, 4) */
ORC_API int64_t orc_s2x_encode(uint8_t *dst, size_t cap, const uint8_t *src, int64_t n, int mode) {
    if (mode != 3 && mode != 4) return orc_s2_encode(dst, cap, src, n, mode);
    int64_t need = orc_s2_max_encoded_len(n);
    if (need < 0) return ORC_ERR_TOO_BIG;
    if ((int64_t)cap < need) return ORC_ERR_DST_SMALL;
    int64_t d = (int64_t)put_uvarint(dst, (uint64_t)n);
    if (n == 0) return d;
    if (n < MIN_NON_LITERAL) return d + orc_s2_emit_literal(dst + d, src, (size_t)n);
    int64_t b = encode_block_best(dst + d, src, n, mode == 4);
    if (b < 0) return b;
    if (b > 0) return d + b;
    return d + orc_s2_emit_literal(dst + d, src, (size_t)n);
}
