/*
 * oracle/orc_flate_nolz.c -- flate.NewWriter(w, level), zlib.NewWriterLevel(w, level) and gzip.NewWriterLevel(w, level)
 * at HuffmanOnly (-2, ConstantCompression) and NoCompression (0) for Writes then Close: a plain-C restatement of exactly
 * the reference code these two levels reach beyond the bit writer.
 *
 * TEST INFRASTRUCTURE ONLY (see orc_common.h); built as its own library by flate_nolz.mk, with -ffp-contract=off.  It
 * compiles orc_deflate.c into the same unit, so the huffmanBitWriter (writeBlockHuff, stored blocks, the reuse state) is
 * that file's, here with logNewTablePenalty 10.  The writer's decision counters stay in orc_deflate_paths; this file's
 * own are in orc_nolz_paths.
 *
 *   flate/deflate.go            writeStoredBlock :354-360, store :683-688, fillBlock :692-696, storeHuff :701-708,
 *                               write :755-770, init (levels 0 and -2) :787-797, close :865-880
 *   zlib/writer.go              writeHeader :95-138 (levels -2, 0 and 1: 78 01), Close :177-195
 *   gzip/gzip.go                XFL :193-198 (0 at these levels; the caller's header blob carries it)
 */
#include "orc_deflate.c"

/* decision paths of this file (NP_* indices into orc_nolz_paths) */
enum { NP_EST_SMALL, NP_EST_LARGE, NP_NEW_OWES_EOB, NP_FINAL_FULL, NP_FINAL_TINY, NP_EMPTY, NP_COUNT };
static int64_t g_np_paths[NP_COUNT];

#define NOLZ_HUFF_WINDOW (32 << 10)
#define NOLZ_TINY 16                                 /* a last window of at most this many bytes counts as tiny */

typedef struct {
    bw_t *w;
    int level;
    uint8_t *window; int32_t windowEnd, windowSize;
    int sync;
} compressorNoLZ;

static void store(compressorNoLZ *d) {                                        /* :683-688 */
    if (d->windowEnd > 0 && (d->windowEnd == MAX_STORE_BLOCK || d->sync)) {
        stored_block(d->w, d->window, (size_t)d->windowEnd, 0);             /* writeStoredBlock :354-360 */
        d->windowEnd = 0;
    }
}
static void storeHuff(compressorNoLZ *d) {                                    /* :701-708 */
    if ((d->windowEnd < d->windowSize && !d->sync) || d->windowEnd == 0) return;
    if (d->sync && d->windowEnd == d->windowSize) g_np_paths[NP_FINAL_FULL]++;
    if (d->sync && d->windowEnd <= NOLZ_TINY) g_np_paths[NP_FINAL_TINY]++;
    const int64_t est0 = g_paths[DP_HUFF_STORED_EST], new0 = g_paths[DP_HUFF_NEW];
    const int owed = d->w->lastHeader > 0;
    writeBlockHuff(d->w, 0, d->window, (size_t)d->windowEnd, d->sync);
    if (g_paths[DP_HUFF_STORED_EST] != est0) g_np_paths[d->windowEnd <= 1024 ? NP_EST_SMALL : NP_EST_LARGE]++;
    if (g_paths[DP_HUFF_NEW] != new0 && owed) g_np_paths[NP_NEW_OWES_EOB]++;
    d->windowEnd = 0;
}
static void step(compressorNoLZ *d) { if (d->level == 0) store(d); else storeHuff(d); }
static void compressorWrite(compressorNoLZ *d, const uint8_t *b, size_t n) {   /* :755-770, fillBlock :692-696 */
    while (n > 0) {
        if (d->windowEnd == d->windowSize || d->sync) step(d);
        size_t k = (size_t)(d->windowSize - d->windowEnd);
        if (k > n) k = n;
        memcpy(d->window + d->windowEnd, b, k);
        d->windowEnd += (int32_t)k;
        b += k; n -= k;
    }
}
static void compressorClose(compressorNoLZ *d) {                               /* :865-880 */
    d->sync = 1;
    step(d);
    writeStoredHeader(d->w, 0, 1);
    bw_flush(d->w);
}

static uint32_t adler32_upd(uint32_t adler, const uint8_t *p, size_t n) {
    uint32_t s1 = adler & 0xffff, s2 = adler >> 16;
    for (size_t i = 0; i < n; i++) { s1 = (s1 + p[i]) % 65521; s2 = (s2 + s1) % 65521; }
    return s2 << 16 | s1;
}

/* One member of the given format (0 raw, 1 zlib, 2 gzip) at level (-2 or 0) as the reference's writer writes it for the
 * Writes in[0, writes[0]), in[writes[0], writes[0] + writes[1]), ... then Close.  hdr: the gzip member header (format 2).
 * check (optional) gets the CRC-32 (raw, gzip) or Adler-32 (zlib) of the input.  Returns the bytes, ORC_ERR_DST_SMALL, or
 * ORC_ERR_SIZE for another level. */
ORC_API int64_t orc_flate_nolz(int level, int format, const uint8_t *hdr, size_t hlen, const uint8_t *in,
                               const size_t *writes, size_t nwrites, uint8_t *out, size_t cap, uint32_t *check) {
    if (level != 0 && level != -2) return ORC_ERR_SIZE;
    size_t total = 0;
    for (size_t k = 0; k < nwrites; k++) total += writes[k];
    compressorNoLZ d;
    memset(&d, 0, sizeof d);
    bw_t *w = malloc(sizeof *w);
    bw_init(w, out, cap);
    d.w = w; d.level = level;
    if (level == 0) {                              /* init :788-791 */
        d.windowSize = MAX_STORE_BLOCK;
    } else {                                       /* :792-796 */
        w->logNewTablePenalty = 10;
        d.windowSize = NOLZ_HUFF_WINDOW;
    }
    d.window = malloc((size_t)d.windowSize);
    if (format == 1) {                             /* zlib writeHeader: 0x78, FLEVEL 0, FCHECK */
        uint8_t h[2] = {0x78, 0 << 6};
        h[1] += (uint8_t)(31 - ((uint32_t)h[0] << 8 | h[1]) % 31);
        writeBytes(w, h, 2);
    } else if (format == 2) {
        writeBytes(w, hdr, hlen);
    }
    if (total == 0) g_np_paths[NP_EMPTY]++;
    const uint8_t *p = in;
    for (size_t k = 0; k < nwrites; k++) { compressorWrite(&d, p, writes[k]); p += writes[k]; }
    compressorClose(&d);
    uint32_t c = format == 1 ? adler32_upd(1, in, total) : crc32_upd(0, in, total);
    if (format == 1) {
        for (int k = 0; k < 4; k++) bw_byte(w, (uint8_t)(c >> (24 - 8 * k)));
    } else if (format == 2) {
        for (int k = 0; k < 4; k++) bw_byte(w, (uint8_t)(c >> (8 * k)));
        for (int k = 0; k < 4; k++) bw_byte(w, (uint8_t)((uint32_t)total >> (8 * k)));
    }
    if (check) *check = c;
    int64_t r = w->overflow ? ORC_ERR_DST_SMALL : (int64_t)w->n;
    free(d.window); free(w);
    return r;
}

/* the decision-path counters (NP_* order), and their reset */
ORC_API void orc_nolz_paths(int64_t *out) { memcpy(out, g_np_paths, sizeof g_np_paths); }
ORC_API void orc_nolz_paths_reset(void) { memset(g_np_paths, 0, sizeof g_np_paths); }
