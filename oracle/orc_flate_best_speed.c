/*
 * oracle/orc_flate_best_speed.c -- flate.NewWriter(w, BestSpeed), zlib.NewWriterLevel(w, BestSpeed) and
 * gzip.NewWriterLevel(w, BestSpeed) for Writes then Close: a plain-C restatement of exactly the reference code that level 1
 * reaches beyond the stateless path.
 *
 * TEST INFRASTRUCTURE ONLY (see orc_common.h); built as its own library by flate_best_speed.mk, with -ffp-contract=off.
 * It compiles orc_deflate.c into the same unit, so the huffmanBitWriter (writeBlockDynamic, writeBlockHuff, stored blocks,
 * the reuse state) is that file's, one restatement for both levels, here with logNewTablePenalty 7.  The writer's decision
 * counters stay in orc_deflate_paths; this file's own are in orc_best_speed_paths.
 *
 *   flate/deflate.go            writeStoredBlock :354-360, storeFast :713-751, write :755-770, init (level 1) :803-808,
 *                               close :865-880
 *   flate/fast_encoder.go       newFastEnc :19-22, hashLen :118-133, addBlock :81-101, Reset :179-189
 *   flate/level1.go             fastEncL1.Encode :18-215
 *   zlib/writer.go              writeHeader :95-138, Write :142-160, Close :177-195
 *   gzip/gzip.go                XFL :193-196 (the caller's header blob carries it)
 */
#include "orc_deflate.c"

/* decision paths of this file (L1P_* indices into orc_best_speed_paths) */
enum { L1P_SF_STORED, L1P_SF_HUFF, L1P_SF_DYN, L1P_SF_FINAL_STORED, L1P_SF_FINAL_HUFF, L1P_PREV_WINDOW, L1P_HIST_MOVE,
       L1P_BACK_STOP, L1P_BACK_STOP_MOVED, L1P_COUNT };
static int64_t g_l1_paths[L1P_COUNT];

/* ---- BestSpeed: fastEncL1 over fastGen's history, and the compressor that drives it */
#define L1_TABLE_BITS 15
#define L1_MAX_MATCH_OFFSET 32768
#define L1_ALLOC_HISTORY (MAX_STORE_BLOCK * 5)
#define L1_BUFFER_RESET ((int32_t)((1u << 31) - 1) - L1_ALLOC_HISTORY - MAX_STORE_BLOCK)
#define L1_MAX_INPUT (1u << 30)

typedef struct {
    uint8_t *hist; int32_t hlen;                 /* e.hist: its bytes and len; cap is L1_ALLOC_HISTORY once allocated */
    int32_t cur;
    int32_t table[1 << L1_TABLE_BITS];
} fastEncL1;

static uint32_t hashLen5(uint64_t u) { return (uint32_t)(((u << 24) * 889523592379ull) >> (64 - L1_TABLE_BITS)); }

static int32_t addBlock(fastEncL1 *e, const uint8_t *src, int32_t n) {         /* fast_encoder.go:81-101 */
    if (e->hist == NULL || e->hlen + n > L1_ALLOC_HISTORY) {
        if (e->hist == NULL) {
            e->hist = malloc(L1_ALLOC_HISTORY + 8);
            e->hlen = 0;
        } else {                                 /* move down the last maxMatchOffset bytes */
            int32_t offset = e->hlen - L1_MAX_MATCH_OFFSET;
            memmove(e->hist, e->hist + offset, L1_MAX_MATCH_OFFSET);
            e->cur += offset;
            e->hlen = L1_MAX_MATCH_OFFSET;
            g_l1_paths[L1P_HIST_MOVE]++;
        }
    }
    int32_t s = e->hlen;
    memcpy(e->hist + e->hlen, src, (size_t)n);
    e->hlen += n;
    return s;
}
static void fastReset(fastEncL1 *e) {                                          /* :179-189 */
    if (e->cur <= L1_BUFFER_RESET) e->cur += L1_MAX_MATCH_OFFSET + e->hlen;
    e->hlen = 0;
}

/* level1.go:18-215.  The table shift at :29-49 needs e.cur >= bufferReset; inputs are at most 1 GiB, so e.cur <=
 * 65 535 + 1 GiB stays below it (see orc_flate_best_speed) and the shift is not restated. */
static void encodeL1(fastEncL1 *e, tokens_t *dst, const uint8_t *in, int32_t n) {
    int32_t s = addBlock(e, in, n);
    if (n < 1 + 1 + 11) { dst->n = (uint32_t)n; return; }    /* never reached from storeFast */
    const uint8_t *src = e->hist;
    const int32_t blockStart = s;
    int32_t nextEmit = s, sLimit = e->hlen - 11;
    uint64_t cv = ld64(src, s);
    for (;;) {
        int32_t nextS, t;
        for (;;) {
            uint32_t nextHash = hashLen5(cv);
            int32_t candidate = e->table[nextHash];
            nextS = s + 2 + ((s - nextEmit) >> 5);
            if (nextS > sLimit) goto emitRemainder;
            uint64_t now = ld64(src, nextS);
            e->table[nextHash] = s + e->cur;
            nextHash = hashLen5(now);
            t = candidate - e->cur;
            if (s - t < L1_MAX_MATCH_OFFSET && (uint32_t)cv == ld32(src, t)) { e->table[nextHash] = nextS + e->cur; break; }
            cv = now;
            s = nextS;
            nextS++;
            candidate = e->table[nextHash];
            now >>= 8;
            e->table[nextHash] = s + e->cur;
            t = candidate - e->cur;
            if (s - t < L1_MAX_MATCH_OFFSET && (uint32_t)cv == ld32(src, t)) { e->table[nextHash] = nextS + e->cur; break; }
            cv = now;
            s = nextS;
        }
        for (;;) {
            int32_t l = matchLen(src + s + 4, src + t + 4, e->hlen - s - 4) + 4;   /* matchlenLong: to the window's end */
            if (t < blockStart) g_l1_paths[L1P_PREV_WINDOW]++;
            while (t > 0 && s > nextEmit && src[t - 1] == src[s - 1]) { s--; t--; l++; }
            if (t == 0 && s > nextEmit) g_l1_paths[e->cur > MAX_STORE_BLOCK ? L1P_BACK_STOP_MOVED : L1P_BACK_STOP]++;
            for (int32_t i = nextEmit; i < s; i++) tok_lit(dst, src[i]);
            tok_match_long(dst, l, (uint32_t)(s - t - 1));                      /* the inlined AddMatchLong */
            s += l;
            nextEmit = s;
            if (nextS >= s) s = nextS + 1;
            if (s >= sLimit) {
                if (s + l + 8 < e->hlen) e->table[hashLen5(ld64(src, s))] = s + e->cur;
                goto emitRemainder;
            }
            uint64_t x = ld64(src, s - 2);
            int32_t o = e->cur + s - 2;
            e->table[hashLen5(x)] = o;
            x >>= 16;
            uint32_t currHash = hashLen5(x);
            int32_t candidate = e->table[currHash];
            e->table[currHash] = o + 2;
            t = candidate - e->cur;
            if (s - t > L1_MAX_MATCH_OFFSET || (uint32_t)x != ld32(src, t)) { cv = x >> 8; s++; break; }
        }
    }
emitRemainder:
    if (nextEmit < e->hlen) {
        if (dst->n == 0) return;
        for (int32_t i = nextEmit; i < e->hlen; i++) tok_lit(dst, src[i]);
    }
}

typedef struct {
    bw_t *w;
    fastEncL1 fast;
    tokens_t tokens;
    uint8_t window[MAX_STORE_BLOCK];
    int32_t windowEnd;
    int sync;
} compressorL1;

static void storeFast(compressorL1 *d) {                                       /* deflate.go:713-751 */
    if (d->windowEnd < MAX_STORE_BLOCK) {
        if (!d->sync) return;
        if (d->windowEnd < 128) {
            if (d->windowEnd == 0) return;
            if (d->windowEnd <= 32) {
                g_l1_paths[L1P_SF_FINAL_STORED]++;
                stored_block(d->w, d->window, (size_t)d->windowEnd, 0);
            } else {
                g_l1_paths[L1P_SF_FINAL_HUFF]++;
                writeBlockHuff(d->w, 0, d->window, (size_t)d->windowEnd, 1);
            }
            tok_reset(&d->tokens);
            d->windowEnd = 0;
            fastReset(&d->fast);
            return;
        }
    }
    encodeL1(&d->fast, &d->tokens, d->window, d->windowEnd);
    if (d->tokens.n == 0) {
        g_l1_paths[L1P_SF_STORED]++;
        stored_block(d->w, d->window, (size_t)d->windowEnd, 0);
    } else if ((int)d->tokens.n > d->windowEnd - (d->windowEnd >> 4)) {
        g_l1_paths[L1P_SF_HUFF]++;
        writeBlockHuff(d->w, 0, d->window, (size_t)d->windowEnd, d->sync);
    } else {
        g_l1_paths[L1P_SF_DYN]++;
        writeBlockDynamic(d->w, &d->tokens, 0, d->window, (size_t)d->windowEnd, d->sync);
    }
    tok_reset(&d->tokens);
    d->windowEnd = 0;
}
static void compressorWrite(compressorL1 *d, const uint8_t *b, size_t n) {   /* :755-770, fillBlock :692-696 */
    while (n > 0) {
        if (d->windowEnd == MAX_STORE_BLOCK || d->sync) storeFast(d);
        size_t k = (size_t)(MAX_STORE_BLOCK - d->windowEnd);
        if (k > n) k = n;
        memcpy(d->window + d->windowEnd, b, k);
        d->windowEnd += (int32_t)k;
        b += k; n -= k;
    }
}
static void compressorClose(compressorL1 *d) {                                 /* :865-880 */
    d->sync = 1;
    storeFast(d);
    writeStoredHeader(d->w, 0, 1);
    bw_flush(d->w);
}

static uint32_t adler32_upd(uint32_t adler, const uint8_t *p, size_t n) {
    uint32_t s1 = adler & 0xffff, s2 = adler >> 16;
    for (size_t i = 0; i < n; i++) { s1 = (s1 + p[i]) % 65521; s2 = (s2 + s1) % 65521; }
    return s2 << 16 | s1;
}

/* One member of the given format (0 raw, 1 zlib, 2 gzip) as the reference's writer at BestSpeed writes it for the Writes
 * in[0, writes[0]), in[writes[0], writes[0] + writes[1]), ... then Close.  hdr: the gzip member header (format 2).  check
 * (optional) gets the CRC-32 (raw, gzip) or Adler-32 (zlib) of the input.  Returns the bytes, ORC_ERR_DST_SMALL, or
 * ORC_ERR_SIZE for more than 1 GiB of input (the device's cap: below it e.cur never reaches bufferReset). */
ORC_API int64_t orc_flate_best_speed(int format, const uint8_t *hdr, size_t hlen, const uint8_t *in, const size_t *writes,
                                     size_t nwrites, uint8_t *out, size_t cap, uint32_t *check) {
    size_t total = 0;
    for (size_t k = 0; k < nwrites; k++) total += writes[k];
    if (total > L1_MAX_INPUT) return ORC_ERR_SIZE;
    compressorL1 *d = calloc(1, sizeof *d);
    bw_t *w = malloc(sizeof *w);
    bw_init(w, out, cap);
    w->logNewTablePenalty = 7;                   /* init, level 1 */
    d->w = w;
    d->fast.cur = MAX_STORE_BLOCK;               /* newFastEnc(1) */
    d->tokens.tokens = malloc((MAX_STORE_BLOCK + 2) * sizeof(uint32_t));
    tok_reset(&d->tokens);
    if (format == 1) {                           /* zlib writeHeader: 0x78, FLEVEL 0, FCHECK */
        uint8_t h[2] = {0x78, 0 << 6};
        h[1] += (uint8_t)(31 - ((uint32_t)h[0] << 8 | h[1]) % 31);
        writeBytes(w, h, 2);
    } else if (format == 2) {
        writeBytes(w, hdr, hlen);
    }
    const uint8_t *p = in;
    for (size_t k = 0; k < nwrites; k++) { compressorWrite(d, p, writes[k]); p += writes[k]; }
    compressorClose(d);
    uint32_t c = format == 1 ? adler32_upd(1, in, total) : crc32_upd(0, in, total);
    if (format == 1) {
        for (int k = 0; k < 4; k++) bw_byte(w, (uint8_t)(c >> (24 - 8 * k)));
    } else if (format == 2) {
        for (int k = 0; k < 4; k++) bw_byte(w, (uint8_t)(c >> (8 * k)));
        for (int k = 0; k < 4; k++) bw_byte(w, (uint8_t)((uint32_t)total >> (8 * k)));
    }
    if (check) *check = c;
    int64_t r = w->overflow ? ORC_ERR_DST_SMALL : (int64_t)w->n;
    free(d->fast.hist); free(d->tokens.tokens); free(d); free(w);
    return r;
}

/* the decision-path counters (L1P_* order), and their reset */
ORC_API void orc_best_speed_paths(int64_t *out) { memcpy(out, g_l1_paths, sizeof g_l1_paths); }
ORC_API void orc_best_speed_paths_reset(void) { memset(g_l1_paths, 0, sizeof g_l1_paths); }
