/*
 * oracle/orc_flate.c -- raw DEFLATE, zlib and gzip decoding: a plain-C restatement of the reference's readers over one
 * whole input (flate.NewReader / zlib.NewReader / gzip.NewReader followed by io.ReadAll).
 *
 * TEST INFRASTRUCTURE ONLY (see orc_common.h); built as its own library by flate.mk.
 *
 *   flate/inflate.go   huffmanDecoder.init :116-279, nextBlock :352-395, readHuffman :464-597, dataBlock :600-646,
 *                      moreBits :728-737, huffSym :740-790; the block decoder of flate/inflate_gen.go :26-270
 *   gzip/gunzip.go     readString :150-179, readHeader :183-253, Read :256-295 (multistream :283-291)
 *   zlib/reader.go     Read :93-121, Reset :134-187
 *
 * The decoder keeps the reference's data structures: the two huffmanDecoders with their chunk and link tables (kept
 * across blocks and gzip members, as flate's Reset keeps h1 and h2), the 32-bit bit buffer filled one byte at a time, and
 * maxRead.  So an empty tree keeps the chunks of the tree that held its slot before (with linkMask cleared), and a symbol
 * is only looked up once maxRead bits are buffered -- both decide outcomes on invalid and truncated streams.
 *
 * Outcomes (orc_flate_decode): the content's byte count, or
 *   ORC_ERR_CORRUPT      flate.CorruptInputError
 *   ORC_FLATE_ERR_EOF    io.ErrUnexpectedEOF; also gzip's io.EOF before the first member's header is complete (an empty
 *                        input, or one that ends inside the first header's name or comment: NewReader fails with io.EOF)
 *   ORC_ERR_MAGIC        gzip.ErrHeader / zlib.ErrHeader
 *   ORC_ERR_CRC          gzip.ErrChecksum / zlib.ErrChecksum
 *   ORC_ERR_UNSUPPORTED  zlib.ErrDictionary (a preset dictionary other than the empty one)
 *   ORC_ERR_DST_SMALL    the content is longer than cap
 * The reference's InternalError("unexpected length code") (inflate.go:531, a code-length symbol above 18 read from a stale
 * table) is reported as ORC_ERR_CORRUPT.
 * Errors are reported in stream order: a checksum that fails ends the read before the next member's first byte.
 * The reference ends a raw DEFLATE stream without error when the input runs out inside the extra bits of a length or a
 * distance (it returns the reader's io.EOF there, inflate_gen.go:121,149,217): the content so far is the result.
 */
#include <stdlib.h>
#include "orc_common.h"

enum { ORC_FLATE_ERR_EOF = -12 };
enum { FL_RAW = 0, FL_ZLIB = 1, FL_GZIP = 2 };
enum { FL_EOF_QUIRK = 1 };   /* internal: the reader's plain io.EOF (see above) */

#define HUFF_CHUNK_BITS 9
#define HUFF_NUM_CHUNKS 512
#define MAX_NUM_LIT 286
#define MAX_NUM_DIST 30
#define NUM_CODES 19

typedef struct {
    int maxRead;
    uint16_t chunks[HUFF_NUM_CHUNKS];
    uint16_t links[HUFF_NUM_CHUNKS][1 << (15 - HUFF_CHUNK_BITS)];
    int nlinks;
    uint32_t linkMask;
} hdec;

static uint16_t rev16(uint16_t v) {
    v = (uint16_t)((v >> 1 & 0x5555) | (v & 0x5555) << 1);
    v = (uint16_t)((v >> 2 & 0x3333) | (v & 0x3333) << 2);
    v = (uint16_t)((v >> 4 & 0x0f0f) | (v & 0x0f0f) << 4);
    return (uint16_t)(v >> 8 | v << 8);
}

/* huffmanDecoder.init, inflate.go:116-279 */
static int hdec_init(hdec *h, const int *lengths, int n) {
    if (h->maxRead != 0) { h->maxRead = 0; h->linkMask = 0; }   /* *h = huffmanDecoder{chunks, links} */
    int count[16] = {0}, min = 0, max = 0;
    for (int i = 0; i < n; i++) {
        const int l = lengths[i];
        if (l == 0) continue;
        if (min == 0 || l < min) min = l;
        if (l > max) max = l;
        count[l & 15]++;
    }
    if (max == 0) return 1;                                     /* empty tree: the chunks stay as they were */
    int code = 0, nextcode[16] = {0};
    for (int i = min; i <= max; i++) {
        code <<= 1;
        nextcode[i & 15] = code;
        code += count[i & 15];
    }
    if (code != 1 << max && !(code == 1 && max == 1)) return 0;
    h->maxRead = min;
    memset(h->chunks, 0, sizeof(h->chunks));
    if (max > HUFF_CHUNK_BITS) {
        const int numLinks = 1 << (max - HUFF_CHUNK_BITS);
        h->linkMask = (uint32_t)(numLinks - 1);
        const int link = nextcode[HUFF_CHUNK_BITS + 1] >> 1;
        h->nlinks = HUFF_NUM_CHUNKS - link;
        for (int j = link; j < HUFF_NUM_CHUNKS; j++) {
            const int reverse = rev16((uint16_t)j) >> (16 - HUFF_CHUNK_BITS);
            const int off = j - link;
            h->chunks[reverse] = (uint16_t)(off << 4 | (HUFF_CHUNK_BITS + 1));
            memset(h->links[off], 0, sizeof(h->links[off]));
        }
    } else {
        h->nlinks = 0;
    }
    for (int i = 0; i < n; i++) {
        const int l = lengths[i];
        if (l == 0) continue;
        const int c = nextcode[l]++;
        const uint16_t chunk = (uint16_t)(i << 4 | l);
        int reverse = rev16((uint16_t)c) >> (16 - l);
        if (l <= HUFF_CHUNK_BITS) {
            for (int off = reverse; off < HUFF_NUM_CHUNKS; off += 1 << l) h->chunks[off] = chunk;
        } else {
            const int j = reverse & (HUFF_NUM_CHUNKS - 1);
            const int value = h->chunks[j] >> 4;
            reverse >>= HUFF_CHUNK_BITS;
            for (int off = reverse; off < (1 << (15 - HUFF_CHUNK_BITS)) && off <= (int)h->linkMask; off += 1 << (l - HUFF_CHUNK_BITS))
                h->links[value][off] = chunk;
        }
    }
    return 1;
}

typedef struct {
    const uint8_t *src; size_t n, pos;     /* the underlying reader */
    uint32_t b; unsigned nb;               /* bit buffer */
    uint8_t *dst; size_t cap, d;           /* the content so far */
    size_t mstart;                         /* first content byte of this member / stream */
    hdec h1, h2, fixed;
    int final;
} inflater;

static int read_byte(inflater *f, uint8_t *c) {
    if (f->pos >= f->n) return 0;
    *c = f->src[f->pos++];
    return 1;
}
/* moreBits with noEOF */
static int more_bits(inflater *f) {
    uint8_t c;
    if (!read_byte(f, &c)) return ORC_FLATE_ERR_EOF;
    f->b |= (uint32_t)c << (f->nb & 31);
    f->nb += 8;
    return 0;
}
/* the loops of inflate_gen.go that return the reader's error unchanged (length / distance extra bits) */
static int need_bits_quirk(inflater *f, unsigned n) {
    while (f->nb < n) {
        uint8_t c;
        if (!read_byte(f, &c)) return FL_EOF_QUIRK;
        f->b |= (uint32_t)c << (f->nb & 31);
        f->nb += 8;
    }
    return 0;
}
/* huffSym, inflate.go:740-790: the symbol, or a negative error */
static int huff_sym(inflater *f, const hdec *h) {
    unsigned n = (unsigned)h->maxRead;
    for (;;) {
        while (f->nb < n) { int r = more_bits(f); if (r) return r; }
        uint16_t chunk = h->chunks[f->b & (HUFF_NUM_CHUNKS - 1)];
        n = chunk & 15;
        if (n > HUFF_CHUNK_BITS) {
            chunk = h->links[chunk >> 4][(f->b >> HUFF_CHUNK_BITS) & h->linkMask];
            n = chunk & 15;
        }
        if (n <= f->nb) {
            if (n == 0) return ORC_ERR_CORRUPT;
            f->b >>= n;
            f->nb -= n;
            return chunk >> 4;
        }
    }
}

static int put_byte(inflater *f, uint8_t v) {
    if (f->d >= f->cap) return ORC_ERR_DST_SMALL;
    f->dst[f->d++] = v;
    return 0;
}

static const int code_order[NUM_CODES] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

/* readHuffman, inflate.go:464-597 */
static int read_huffman(inflater *f) {
    int bits[MAX_NUM_LIT + MAX_NUM_DIST + 2], codebits[NUM_CODES];
    while (f->nb < 14) { int r = more_bits(f); if (r) return r; }
    const int nlit = (int)(f->b & 0x1f) + 257;
    if (nlit > MAX_NUM_LIT) return ORC_ERR_CORRUPT;
    f->b >>= 5;
    const int ndist = (int)(f->b & 0x1f) + 1;
    if (ndist > MAX_NUM_DIST) return ORC_ERR_CORRUPT;
    f->b >>= 5;
    const int nclen = (int)(f->b & 0xf) + 4;
    f->b >>= 4;
    f->nb -= 14;
    for (int i = 0; i < nclen; i++) {
        while (f->nb < 3) { int r = more_bits(f); if (r) return r; }
        codebits[code_order[i]] = (int)(f->b & 7);
        f->b >>= 3;
        f->nb -= 3;
    }
    for (int i = nclen; i < NUM_CODES; i++) codebits[code_order[i]] = 0;
    if (!hdec_init(&f->h1, codebits, NUM_CODES)) return ORC_ERR_CORRUPT;
    for (int i = 0, n = nlit + ndist; i < n;) {
        const int x = huff_sym(f, &f->h1);
        if (x < 0) return x;
        if (x < 16) { bits[i++] = x; continue; }
        int rep, b;
        unsigned nb;
        if (x == 16) {
            rep = 3; nb = 2;
            if (i == 0) return ORC_ERR_CORRUPT;
            b = bits[i - 1];
        } else if (x == 17) { rep = 3; nb = 3; b = 0; }
        else if (x == 18) { rep = 11; nb = 7; b = 0; }
        else return ORC_ERR_CORRUPT;   /* InternalError("unexpected length code"), inflate.go:531: h1 left stale by an empty code */
        while (f->nb < nb) { int r = more_bits(f); if (r) return r; }
        rep += (int)(f->b & ((1u << nb) - 1));
        f->b >>= nb;
        f->nb -= nb;
        if (i + rep > n) return ORC_ERR_CORRUPT;
        for (int j = 0; j < rep; j++) bits[i++] = b;
    }
    if (!hdec_init(&f->h1, bits, nlit) || !hdec_init(&f->h2, bits + nlit, ndist)) return ORC_ERR_CORRUPT;
    if (f->h1.maxRead < bits[256]) f->h1.maxRead = bits[256];
    if (!f->final) f->h1.maxRead += 10;
    return 0;
}

static const uint8_t len_extra[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
static const uint16_t len_base[29] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115,
                                      131, 163, 195, 227, 258};

/* the block decoder, inflate_gen.go:26-270 (hd == NULL: fixed distance codes) */
static int huffman_block(inflater *f, const hdec *hl, const hdec *hd) {
    for (;;) {
        const int v = huff_sym(f, hl);
        if (v < 0) return v;
        if (v < 256) { int r = put_byte(f, (uint8_t)v); if (r) return r; continue; }
        if (v == 256) return 0;
        if (v >= MAX_NUM_LIT) return ORC_ERR_CORRUPT;
        int length = len_base[v - 257];
        const unsigned ne = len_extra[v - 257];
        if (ne) {
            if (need_bits_quirk(f, ne)) return FL_EOF_QUIRK;
            length += (int)(f->b & ((1u << ne) - 1));
            f->b >>= ne;
            f->nb -= ne;
        }
        uint32_t dist;
        if (!hd) {
            if (need_bits_quirk(f, 5)) return FL_EOF_QUIRK;
            dist = (uint32_t)(rev16((uint16_t)((f->b & 0x1f) << 3)) >> 8);
            f->b >>= 5;
            f->nb -= 5;
        } else {
            const int x = huff_sym(f, hd);
            if (x < 0) return x;
            dist = (uint32_t)x;
        }
        if (dist < 4) dist++;
        else if (dist < MAX_NUM_DIST) {
            const unsigned nb = (dist - 2) >> 1;
            uint32_t extra = (dist & 1) << nb;
            if (need_bits_quirk(f, nb)) return FL_EOF_QUIRK;
            extra |= f->b & ((1u << nb) - 1);
            f->b >>= nb;
            f->nb -= nb;
            dist = (1u << (nb + 1)) + 1 + extra;
        } else return ORC_ERR_CORRUPT;
        if (dist > f->d - f->mstart) return ORC_ERR_CORRUPT;   /* dist > dict.histSize() (dist <= 32768 = the window) */
        for (int k = 0; k < length; k++) {
            if (f->d >= f->cap) return ORC_ERR_DST_SMALL;
            f->dst[f->d] = f->dst[f->d - dist];
            f->d++;
        }
    }
}

/* one DEFLATE stream from f->pos: 0 at its end, FL_EOF_QUIRK, or a negative error */
static int inflate_stream(inflater *f) {
    f->b = 0; f->nb = 0; f->final = 0;
    f->mstart = f->d;
    for (;;) {
        while (f->nb < 3) { int r = more_bits(f); if (r) return r; }
        f->final = f->b & 1;
        const uint32_t typ = (f->b >> 1) & 3;
        f->b >>= 3;
        f->nb -= 3;
        int r;
        if (typ == 0) {                                         /* dataBlock, inflate.go:600-646 */
            const unsigned left = f->nb & 7;
            f->nb -= left; f->b >>= left;
            uint8_t buf[4];
            unsigned have = f->nb >> 3;
            for (unsigned i = 0; i < have; i++) buf[i] = (uint8_t)(f->b >> (8 * i));
            f->nb = 0; f->b = 0;
            for (; have < 4; have++) if (!read_byte(f, &buf[have])) return ORC_FLATE_ERR_EOF;
            const uint16_t n = (uint16_t)(buf[0] | buf[1] << 8), nn = (uint16_t)(buf[2] | buf[3] << 8);
            if (nn != (uint16_t)~n) return ORC_ERR_CORRUPT;
            for (unsigned i = 0; i < n; i++) {
                uint8_t c;
                if (!read_byte(f, &c)) return ORC_FLATE_ERR_EOF;
                if ((r = put_byte(f, c))) return r;
            }
            r = 0;
        } else if (typ == 1) r = huffman_block(f, &f->fixed, NULL);
        else if (typ == 2) {
            if ((r = read_huffman(f))) return r;
            r = huffman_block(f, &f->h1, &f->h2);
        } else return ORC_ERR_CORRUPT;
        if (r) return r;
        if (f->final) return 0;
    }
}

static uint32_t crc32_ieee(uint32_t crc, const uint8_t *p, size_t n) {
    crc = ~crc;
    for (size_t i = 0; i < n; i++) {
        crc ^= p[i];
        for (int k = 0; k < 8; k++) crc = (crc & 1) ? (crc >> 1) ^ 0xedb88320u : crc >> 1;
    }
    return ~crc;
}
static uint32_t adler32(const uint8_t *p, size_t n) {
    uint32_t a = 1, b = 0;
    for (size_t i = 0; i < n; i++) { a = (a + p[i]) % 65521; b = (b + a) % 65521; }
    return b << 16 | a;
}

/* gzip readHeader, gunzip.go:183-253: 0, FL_EOF_QUIRK (the reader's io.EOF) or a negative error */
static int gzip_header(inflater *f) {
    const size_t start = f->pos;
    if (f->n - f->pos < 10) {
        const int none = f->pos == f->n;
        f->pos = f->n;
        return none ? FL_EOF_QUIRK : ORC_FLATE_ERR_EOF;
    }
    const uint8_t *h = f->src + f->pos;
    if (h[0] != 0x1f || h[1] != 0x8b || h[2] != 8) return ORC_ERR_MAGIC;
    const uint8_t flg = h[3];
    f->pos += 10;
    if (flg & 4) {                                              /* FEXTRA */
        if (f->n - f->pos < 2) return ORC_FLATE_ERR_EOF;
        const size_t xlen = (size_t)f->src[f->pos] | (size_t)f->src[f->pos + 1] << 8;
        f->pos += 2;
        if (f->n - f->pos < xlen) return ORC_FLATE_ERR_EOF;
        f->pos += xlen;
    }
    for (int k = 0; k < 2; k++) {                               /* FNAME, FCOMMENT: readString, gunzip.go:150-179 */
        if (!(flg & (k == 0 ? 8 : 16))) continue;
        for (int i = 0;; i++) {
            if (i >= 512) return ORC_ERR_MAGIC;
            uint8_t c;
            if (!read_byte(f, &c)) return FL_EOF_QUIRK;
            if (c == 0) break;
        }
    }
    if (flg & 2) {                                              /* FHCRC */
        if (f->n - f->pos < 2) return ORC_FLATE_ERR_EOF;
        const uint16_t want = (uint16_t)(f->src[f->pos] | f->src[f->pos + 1] << 8);
        if (want != (uint16_t)crc32_ieee(0, f->src + start, f->pos - start)) return ORC_ERR_MAGIC;
        f->pos += 2;
    }
    if (flg >> 5) return ORC_ERR_MAGIC;
    return 0;
}

ORC_API int64_t orc_flate_decode(int format, int multistream, const uint8_t *src, size_t n, uint8_t *dst, size_t cap) {
    inflater *f = (inflater *)calloc(1, sizeof(inflater));
    if (!f) return ORC_ERR_INTERNAL;
    f->src = src; f->n = n; f->dst = dst; f->cap = cap;
    {   /* fixedHuffmanDecoderInit, inflate.go:65-90 */
        int bits[288];
        for (int i = 0; i < 144; i++) bits[i] = 8;
        for (int i = 144; i < 256; i++) bits[i] = 9;
        for (int i = 256; i < 280; i++) bits[i] = 7;
        for (int i = 280; i < 288; i++) bits[i] = 8;
        hdec_init(&f->fixed, bits, 288);
    }
    int64_t res;
    int r;
    if (format == FL_RAW) {
        r = inflate_stream(f);
        res = r < 0 ? r : (int64_t)f->d;                        /* (FL_EOF_QUIRK included) */
    } else if (format == FL_ZLIB) {
        res = 0;
        if (n < 2) res = ORC_FLATE_ERR_EOF;
        else if ((src[0] & 15) != 8 || (src[0] >> 4) > 7 || (((unsigned)src[0] << 8 | src[1]) % 31) != 0) res = ORC_ERR_MAGIC;
        else {
            f->pos = 2;
            if (src[1] & 0x20) {
                if (n < 6) res = ORC_FLATE_ERR_EOF;
                else if (((uint32_t)src[2] << 24 | (uint32_t)src[3] << 16 | (uint32_t)src[4] << 8 | src[5]) != 1) res = ORC_ERR_UNSUPPORTED;
                f->pos = 6;                                     /* adler32 of the empty dictionary: decoded without one */
            }
        }
        if (res == 0) {
            r = inflate_stream(f);
            if (r < 0) res = r;
            else if (f->n - f->pos < 4)                         /* (FL_EOF_QUIRK: the input is used up) */ res = ORC_FLATE_ERR_EOF;
            else {
                const uint8_t *t = src + f->pos;
                const uint32_t want = (uint32_t)t[0] << 24 | (uint32_t)t[1] << 16 | (uint32_t)t[2] << 8 | t[3];
                res = want == adler32(dst, f->d) ? (int64_t)f->d : ORC_ERR_CRC;
            }
        }
    } else {
        r = gzip_header(f);
        res = r == FL_EOF_QUIRK ? ORC_FLATE_ERR_EOF : r;
        while (res == 0) {
            r = inflate_stream(f);
            if (r < 0) { res = r; break; }
            if (f->n - f->pos < 8)                              /* (FL_EOF_QUIRK: the input is used up) */ { res = ORC_FLATE_ERR_EOF; break; }
            const uint8_t *t = src + f->pos;
            const uint32_t crc = (uint32_t)t[0] | (uint32_t)t[1] << 8 | (uint32_t)t[2] << 16 | (uint32_t)t[3] << 24;
            const uint32_t isz = (uint32_t)t[4] | (uint32_t)t[5] << 8 | (uint32_t)t[6] << 16 | (uint32_t)t[7] << 24;
            f->pos += 8;
            if (crc != crc32_ieee(0, dst + f->mstart, f->d - f->mstart) || isz != (uint32_t)(f->d - f->mstart)) { res = ORC_ERR_CRC; break; }
            if (!multistream) break;
            r = gzip_header(f);
            if (r == FL_EOF_QUIRK) break;                       /* io.EOF: the end of the members */
            if (r) { res = r; break; }
        }
        if (res == 0) res = (int64_t)f->d;
    }
    free(f);
    return res;
}
