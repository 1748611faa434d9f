/*
 * oracle/orc_deflate.c -- flate.StatelessDeflate and the gzip framing of gzip.NewWriterLevel(w, StatelessCompression):
 * a plain-C restatement of exactly the reference code the stateless path reaches.
 *
 * TEST INFRASTRUCTURE ONLY (see orc_common.h); built as its own library by deflate.mk, with -ffp-contract=off: the
 * reference's float32 / float64 decisions are reproduced operation by operation, as Go computes them on amd64.
 *
 *   flate/stateless.go          StatelessDeflate :76-162, hashSL :164-166, statelessEnc :176-325
 *   flate/token.go              mFastLog2 :212-220, EstimatedBits :225-260, AddMatchLong :284-309, AddEOB :311-315,
 *                               offsetCode :365-379
 *   flate/huffman_code.go       bitLength :132-140, canReuseBits :151-163, bitCounts :183-309,
 *                               assignEncodingAndSize :313-333, generate :339-371, atLeastOne :374-382
 *   flate/huffman_bit_writer.go canReuse :163-190, flush :192-218, generateCodegen :269-348, codegens / headerSize
 *                               :350-368, dynamicReuseSize / dynamicSize / extraBitSize / fixedSize / storedSize :371-419,
 *                               writeDynamicHeader :458-497, writeStoredHeader :502-529, writeFixedHeader :531-547,
 *                               writeBlockDynamic :620-765, indexTokens :784-815, writeTokens :824-971,
 *                               huffOffset :975-982, writeBlockHuff :987-1174
 *   flate/matchlen_generic.go   matchLen :14-35
 *   gzip/gzip.go                Write :171-235, Close :264-290
 *
 * The bit writer's 48-bit staging and its 246-byte buffer only batch the stream: the output is the sequence of codes
 * written, so here bits go straight to the output.  sortByFreq / sortByLiteral order by a total key (literals are
 * distinct), so any sort gives the reference's order.  A pooled huffmanBitWriter starts every StatelessDeflate call with
 * lastHeader 0 and logNewTablePenalty 0, so nothing carries between calls.
 */
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include "orc_common.h"

#define LITERAL_COUNT 286
#define OFFSET_CODE_COUNT 30
#define END_BLOCK 256
#define CODEGEN_COUNT 19
#define BAD_CODE 255
#define MAX_PREDEFINED_TOKENS 250
#define MAX_STORE_BLOCK 65535
#define MATCH_TYPE (1u << 30)
#define LENGTH_SHIFT 22
#define MAX_STATELESS_BLOCK 32767
#define MAX_STATELESS_DICT (8 << 10)

/* decision paths, counted for the tests (dp_* indices into orc_deflate_paths) */
enum { DP_STORED_EMPTY_TOKENS, DP_HUFF_STORED_TEST, DP_HUFF_STORED_EST, DP_HUFF_NEW, DP_HUFF_REUSE, DP_DYN_NEW,
       DP_DYN_REUSE, DP_DYN_FIXED, DP_DYN_STORED, DP_EOB_BEFORE_STORED, DP_LONG_MATCH, DP_COUNT };
static int64_t g_paths[DP_COUNT];

static const uint8_t lengthExtraBits[32] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5,
                                            5, 5, 0};
static const uint8_t lengthBase[32] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 10, 12, 14, 16, 20, 24, 28, 32, 40, 48, 56, 64, 80, 96,
                                       112, 128, 160, 192, 224, 255};
static const int8_t offsetExtraBits[32] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11,
                                           11, 12, 12, 13, 13, 14, 14};
static const uint32_t offsetBase[32] = {0x000000, 0x000001, 0x000002, 0x000003, 0x000004, 0x000006, 0x000008, 0x00000c,
                                        0x000010, 0x000018, 0x000020, 0x000030, 0x000040, 0x000060, 0x000080, 0x0000c0,
                                        0x000100, 0x000180, 0x000200, 0x000300, 0x000400, 0x000600, 0x000800, 0x000c00,
                                        0x001000, 0x001800, 0x002000, 0x003000, 0x004000, 0x006000};
static const uint32_t codegenOrder[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

/* lengthCodes[len] (token.go:30-57) for len = length - 3 in [0, 255]: the code whose range holds len, 255 -> 28 */
static uint8_t lengthCode(uint32_t len) {
    uint8_t c = 0;
    while (c < 28 && lengthBase[c + 1] <= len) c++;
    return c;
}
static uint32_t offsetCode(uint32_t off) {     /* token.go:365-379 (off < 32768) */
    if (off < 4) return off;
    uint32_t hb = 31 - (uint32_t)__builtin_clz(off);
    return 2 * hb + ((off >> (hb - 1)) & 1);
}

/* ---- tokens (token.go) */
typedef struct {
    uint16_t extraHist[32], offHist[32], litHist[256];
    uint32_t n;
    uint32_t *tokens;
} tokens_t;

static void tok_reset(tokens_t *t) {
    t->n = 0;
    memset(t->extraHist, 0, sizeof t->extraHist); memset(t->offHist, 0, sizeof t->offHist);
    memset(t->litHist, 0, sizeof t->litHist);
}
static void tok_lit(tokens_t *t, uint8_t v) { t->tokens[t->n++] = v; t->litHist[v]++; }
static void tok_match_long(tokens_t *t, int32_t xlength, uint32_t xoffset) {    /* AddMatchLong :284-309 */
    uint32_t oc = offsetCode(xoffset);
    xoffset |= oc << 16;
    if (xlength > 258) g_paths[DP_LONG_MATCH]++;
    while (xlength > 0) {
        int32_t xl = xlength;
        if (xl > 258) xl = xl > 258 + 3 ? 258 : 258 - 3;
        xlength -= xl;
        xl -= 3;
        t->extraHist[lengthCode((uint8_t)xl) + 1]++;
        t->offHist[oc & 31]++;
        t->tokens[t->n++] = MATCH_TYPE | (uint32_t)xl << LENGTH_SHIFT | xoffset;
    }
}
static void tok_match(tokens_t *t, uint32_t xlength, uint32_t xoffset) {      /* AddMatch :264-280 */
    uint32_t oc = offsetCode(xoffset);
    xoffset |= oc << 16;
    t->extraHist[lengthCode((uint8_t)xlength) + 1]++;
    t->offHist[oc & 31]++;
    t->tokens[t->n++] = MATCH_TYPE | xlength << LENGTH_SHIFT | xoffset;
}
static void tok_eob(tokens_t *t) { t->tokens[t->n++] = END_BLOCK; t->extraHist[0]++; }

static float f32frombits(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }
static uint32_t f32bits(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }
static float mFastLog2(float val) {                                             /* :212-220 */
    int32_t ux = (int32_t)f32bits(val);
    float log2 = (float)(((ux >> 23) & 255) - 128);
    ux &= -0x7f800001;
    ux += 127 << 23;
    float uval = f32frombits((uint32_t)ux);
    float a = -0.34484843f * uval;
    a = a + 2.02466578f;
    a = a * uval;
    a = a - 0.67487759f;
    log2 += a;
    return log2;
}
static float atLeastOne(float v) { return v < 1 ? 1 : (v > 15 ? 15 : v); }
static int estimatedBits(const tokens_t *t) {                                  /* :225-260 (nFilled is 0) */
    float shannon = 0;
    int bits = 0, nMatches = 0, total = (int)t->n;
    if (total > 0) {
        float invTotal = 1.0f / (float)total;
        for (int i = 0; i < 256; i++) {
            if (t->litHist[i]) {
                float n = (float)t->litHist[i];
                shannon += atLeastOne(-mFastLog2(n * invTotal)) * n;
            }
        }
        shannon += 15;
        for (int i = 0; i < 29; i++) {
            uint16_t v = t->extraHist[1 + i];
            if (v) {
                float n = (float)v;
                shannon += atLeastOne(-mFastLog2(n * invTotal)) * n;
                bits += lengthExtraBits[i & 31] * (int)v;
                nMatches += v;
            }
        }
    }
    if (nMatches > 0) {
        float invTotal = 1.0f / (float)nMatches;
        for (int i = 0; i < OFFSET_CODE_COUNT; i++) {
            uint16_t v = t->offHist[i];
            if (v) {
                float n = (float)v;
                shannon += atLeastOne(-mFastLog2(n * invTotal)) * n;
                bits += offsetExtraBits[i & 31] * (int)v;
            }
        }
    }
    return (int)shannon + bits;
}

/* ---- huffmanEncoder (huffman_code.go); hcode = len | code << 8 */
typedef struct { uint32_t codes[320]; int32_t bitCount[17]; } henc;
typedef struct { uint16_t literal, freq; } lnode;

static uint16_t rev16(uint16_t v) {
    v = (uint16_t)((v >> 1 & 0x5555) | (v & 0x5555) << 1);
    v = (uint16_t)((v >> 2 & 0x3333) | (v & 0x3333) << 2);
    v = (uint16_t)((v >> 4 & 0x0f0f) | (v & 0x0f0f) << 4);
    return (uint16_t)(v >> 8 | v << 8);
}
static uint32_t newhcode(uint16_t code, uint8_t len) { return len | (uint32_t)code << 8; }
static uint16_t reverseBits(uint16_t number, uint8_t bitLength) { return rev16((uint16_t)(number << ((16 - bitLength) & 15))); }
static int hlen(uint32_t h) { return h & 0xff; }

static int henc_bitLength(const henc *h, const uint16_t *freq, int n) {
    int total = 0;
    for (int i = 0; i < n; i++) if (freq[i]) total += freq[i] * hlen(h->codes[i]);
    return total;
}
static int henc_canReuseBits(const henc *h, const uint16_t *freq, int n) {
    int total = 0;
    for (int i = 0; i < n; i++) {
        if (freq[i]) {
            if (h->codes[i] == 0) return 0x7fffffff;
            total += freq[i] * hlen(h->codes[i]);
        }
    }
    return total;
}
static int cmp_freq(const void *a, const void *b) {
    const lnode *x = a, *y = b;
    if (x->freq != y->freq) return x->freq < y->freq ? -1 : 1;
    return x->literal < y->literal ? -1 : (x->literal > y->literal);
}
static int cmp_lit(const void *a, const void *b) {
    const lnode *x = a, *y = b;
    return x->literal < y->literal ? -1 : (x->literal > y->literal);
}
typedef struct { int32_t level, lastFreq, nextCharFreq, nextPairFreq, needed; } levelInfo;

static void bitCounts(henc *h, lnode *list, int32_t n, int32_t maxBits) {      /* :183-309 */
    list[n].literal = 0xffff; list[n].freq = 0xffff;
    if (maxBits > n - 1) maxBits = n - 1;
    levelInfo levels[16];
    int32_t leafCounts[16][16];
    memset(levels, 0, sizeof levels); memset(leafCounts, 0, sizeof leafCounts);
    int32_t l2f = list[2].freq, l1f = list[1].freq, l0f = (int32_t)list[0].freq + list[1].freq;
    for (int32_t level = 1; level <= maxBits; level++) {
        levels[level] = (levelInfo){level, l1f, l2f, l0f, 0};
        leafCounts[level][level] = 2;
        if (level == 1) levels[level].nextPairFreq = 0x7fffffff;
    }
    levels[maxBits].needed = 2 * n - 4;
    uint32_t level = (uint32_t)maxBits;
    while (level < 16) {
        levelInfo *l = &levels[level];
        if (l->nextPairFreq == 0x7fffffff && l->nextCharFreq == 0x7fffffff) {
            l->needed = 0;
            levels[level + 1].nextPairFreq = 0x7fffffff;
            level++;
            continue;
        }
        int32_t prevFreq = l->lastFreq;
        if (l->nextCharFreq < l->nextPairFreq) {
            int32_t nn = leafCounts[level][level] + 1;
            l->lastFreq = l->nextCharFreq;
            leafCounts[level][level] = nn;
            lnode e = list[nn];
            l->nextCharFreq = e.literal < 0xffff ? (int32_t)e.freq : 0x7fffffff;
        } else {
            l->lastFreq = l->nextPairFreq;
            int32_t save = leafCounts[level][level];
            memcpy(leafCounts[level], leafCounts[level - 1], sizeof leafCounts[level]);
            leafCounts[level][level] = save;
            levels[l->level - 1].needed = 2;
        }
        if (--l->needed == 0) {
            if (l->level == maxBits) break;
            levels[l->level + 1].nextPairFreq = prevFreq + l->lastFreq;
            level++;
        } else {
            while (levels[level - 1].needed > 0) level--;
        }
    }
    int bits = 1;
    for (int32_t lv = maxBits; lv > 0; lv--) {
        h->bitCount[bits] = leafCounts[maxBits][lv] - leafCounts[maxBits][lv - 1];
        bits++;
    }
    h->bitCount[0] = 0;
    for (int i = maxBits + 1; i < 17; i++) h->bitCount[i] = -1;   /* bitCount is sliced to maxBits + 1 */
}
static void assignEncodingAndSize(henc *h, lnode *list, int32_t len) {         /* :313-333 */
    uint16_t code = 0;
    for (int n = 0; n < 17 && h->bitCount[n] >= 0; n++) {
        int32_t bits = h->bitCount[n];
        code <<= 1;
        if (n == 0 || bits == 0) continue;
        lnode *chunk = list + len - bits;
        qsort(chunk, (size_t)bits, sizeof(lnode), cmp_lit);
        for (int i = 0; i < bits; i++) {
            h->codes[chunk[i].literal] = newhcode(reverseBits(code, (uint8_t)n), (uint8_t)n);
            code++;
        }
        len -= bits;
    }
}
static void henc_generate(henc *h, const uint16_t *freq, int nfreq, int32_t maxBits) {  /* :339-371 */
    lnode list[LITERAL_COUNT + 1];
    int count = 0;
    for (int i = 0; i < nfreq; i++) {
        if (freq[i]) { list[count].literal = (uint16_t)i; list[count].freq = freq[i]; count++; }
        else h->codes[i] = 0;
    }
    if (count <= 2) {
        for (int i = 0; i < count; i++) h->codes[list[i].literal] = newhcode((uint16_t)i, 1);
        return;
    }
    qsort(list, (size_t)count, sizeof(lnode), cmp_freq);
    bitCounts(h, list, count, maxBits);
    assignEncodingAndSize(h, list, count);
}

static henc fixedLit, fixedOff, huffOffset;
static void init_fixed(void) {
    static int done;
    if (done) return;
    for (int ch = 0; ch < LITERAL_COUNT; ch++) {
        uint16_t bits; uint8_t size;
        if (ch < 144) { bits = (uint16_t)(ch + 48); size = 8; }
        else if (ch < 256) { bits = (uint16_t)(ch + 400 - 144); size = 9; }
        else if (ch < 280) { bits = (uint16_t)(ch - 256); size = 7; }
        else { bits = (uint16_t)(ch + 192 - 280); size = 8; }
        fixedLit.codes[ch] = newhcode(reverseBits(bits, size), size);
    }
    for (int ch = 0; ch < 30; ch++) fixedOff.codes[ch] = newhcode(reverseBits((uint16_t)ch, 5), 5);
    uint16_t f[OFFSET_CODE_COUNT] = {1};
    henc_generate(&huffOffset, f, OFFSET_CODE_COUNT, 15);
    done = 1;
}

/* ---- huffmanBitWriter */
typedef struct {
    uint8_t *out; size_t cap, n; int overflow;
    uint64_t bits; unsigned nbits;
    int lastHuffMan, lastHeader;
    unsigned logNewTablePenalty;
    henc *literalEncoding, *tmpLitEncoding, offsetEncoding, codegenEncoding;
    henc lit_a, lit_b;
    uint16_t literalFreq[257 + 32], offsetFreq[32], codegenFreq[CODEGEN_COUNT];
    uint8_t codegen[LITERAL_COUNT + OFFSET_CODE_COUNT + 1];
} bw_t;

static void bw_init(bw_t *w, uint8_t *out, size_t cap) {
    memset(w, 0, sizeof *w);
    w->out = out; w->cap = cap;
    w->literalEncoding = &w->lit_a; w->tmpLitEncoding = &w->lit_b;
    init_fixed();
}
static void bw_byte(bw_t *w, uint8_t b) {
    if (w->n < w->cap) w->out[w->n] = b; else w->overflow = 1;
    w->n++;
}
static void writeBits(bw_t *w, uint32_t b, unsigned nb) {
    w->bits |= (uint64_t)b << w->nbits;
    w->nbits += nb;
    while (w->nbits >= 8) { bw_byte(w, (uint8_t)w->bits); w->bits >>= 8; w->nbits -= 8; }
}
static void writeCode(bw_t *w, uint32_t c) { writeBits(w, c >> 8, c & 0xff); }
static void bw_flush(bw_t *w) {                                                /* :192-218 */
    if (w->lastHeader > 0) { writeCode(w, w->literalEncoding->codes[END_BLOCK]); w->lastHeader = 0; }
    if (w->nbits) { bw_byte(w, (uint8_t)w->bits); w->bits = 0; w->nbits = 0; }
}
static void writeBytes(bw_t *w, const uint8_t *p, size_t n) { for (size_t i = 0; i < n; i++) bw_byte(w, p[i]); }

static void generateCodegen(bw_t *w, int numLiterals, int numOffsets, const henc *litEnc, const henc *offEnc) {
    memset(w->codegenFreq, 0, sizeof w->codegenFreq);
    uint8_t *codegen = w->codegen;
    for (int i = 0; i < numLiterals; i++) codegen[i] = (uint8_t)hlen(litEnc->codes[i]);
    for (int i = 0; i < numOffsets; i++) codegen[numLiterals + i] = (uint8_t)hlen(offEnc->codes[i]);
    codegen[numLiterals + numOffsets] = BAD_CODE;
    uint8_t size = codegen[0];
    int count = 1, outIndex = 0;
    for (int inIndex = 1; size != BAD_CODE; inIndex++) {
        uint8_t nextSize = codegen[inIndex];
        if (nextSize == size) { count++; continue; }
        if (size != 0) {
            codegen[outIndex++] = size;
            w->codegenFreq[size]++;
            count--;
            while (count >= 3) {
                int n = count < 6 ? count : 6;
                codegen[outIndex++] = 16; codegen[outIndex++] = (uint8_t)(n - 3);
                w->codegenFreq[16]++;
                count -= n;
            }
        } else {
            while (count >= 11) {
                int n = count < 138 ? count : 138;
                codegen[outIndex++] = 18; codegen[outIndex++] = (uint8_t)(n - 11);
                w->codegenFreq[18]++;
                count -= n;
            }
            if (count >= 3) {
                codegen[outIndex++] = 17; codegen[outIndex++] = (uint8_t)(count - 3);
                w->codegenFreq[17]++;
                count = 0;
            }
        }
        count--;
        for (; count >= 0; count--) { codegen[outIndex++] = size; w->codegenFreq[size]++; }
        size = nextSize;
        count = 1;
    }
    codegen[outIndex] = BAD_CODE;
}
static int codegens(const bw_t *w) {
    int n = CODEGEN_COUNT;
    while (n > 4 && w->codegenFreq[codegenOrder[n - 1]] == 0) n--;
    return n;
}
static int headerSize(const bw_t *w) {
    return 3 + 5 + 5 + 4 + 3 * codegens(w) + henc_bitLength(&w->codegenEncoding, w->codegenFreq, CODEGEN_COUNT) +
           w->codegenFreq[16] * 2 + w->codegenFreq[17] * 3 + w->codegenFreq[18] * 7;
}
static int dynamicReuseSize(const bw_t *w, const henc *litEnc, const henc *offEnc) {
    return henc_bitLength(litEnc, w->literalFreq, 289) + henc_bitLength(offEnc, w->offsetFreq, 32);
}
static int dynamicSize(const bw_t *w, const henc *litEnc, const henc *offEnc, int extraBits) {
    return headerSize(w) + henc_bitLength(litEnc, w->literalFreq, 289) + henc_bitLength(offEnc, w->offsetFreq, 32) + extraBits;
}
static int extraBitSize(const bw_t *w) {
    int total = 0;
    for (int i = 0; i < LITERAL_COUNT - 257; i++) total += w->literalFreq[257 + i] * lengthExtraBits[i & 31];
    for (int i = 0; i < OFFSET_CODE_COUNT; i++) total += w->offsetFreq[i] * offsetExtraBits[i & 31];
    return total;
}
static int fixedSize(const bw_t *w, int extraBits) {
    return 3 + henc_bitLength(&fixedLit, w->literalFreq, 289) + henc_bitLength(&fixedOff, w->offsetFreq, 32) + extraBits;
}
static int storedSize(const uint8_t *in, size_t n, int *storable) {
    *storable = in != NULL && n <= MAX_STORE_BLOCK;
    return *storable ? (int)(n + 5) * 8 : 0;
}
static void writeDynamicHeader(bw_t *w, int numLiterals, int numOffsets, int numCodegens, int isEof) {
    writeBits(w, isEof ? 5 : 4, 3);
    writeBits(w, (uint32_t)(numLiterals - 257), 5);
    writeBits(w, (uint32_t)(numOffsets - 1), 5);
    writeBits(w, (uint32_t)(numCodegens - 4), 4);
    for (int i = 0; i < numCodegens; i++) writeBits(w, (uint32_t)hlen(w->codegenEncoding.codes[codegenOrder[i]]), 3);
    for (int i = 0;;) {
        uint32_t cw = w->codegen[i++];
        if (cw == BAD_CODE) break;
        writeCode(w, w->codegenEncoding.codes[cw]);
        if (cw == 16) writeBits(w, w->codegen[i++], 2);
        else if (cw == 17) writeBits(w, w->codegen[i++], 3);
        else if (cw == 18) writeBits(w, w->codegen[i++], 7);
    }
}
static void writeFixedHeader(bw_t *w, int isEof) {
    if (w->lastHeader > 0) { writeCode(w, w->literalEncoding->codes[END_BLOCK]); w->lastHeader = 0; }
    writeBits(w, isEof ? 3 : 2, 3);
}
static void writeStoredHeader(bw_t *w, int length, int isEof) {
    if (w->lastHeader > 0) {
        writeCode(w, w->literalEncoding->codes[END_BLOCK]); w->lastHeader = 0;
        if (length > 0) g_paths[DP_EOB_BEFORE_STORED]++;
    }
    if (length == 0 && isEof) {
        writeFixedHeader(w, isEof);
        writeBits(w, 0, 7);
        bw_flush(w);
        return;
    }
    writeBits(w, isEof ? 1 : 0, 3);
    bw_flush(w);
    writeBits(w, (uint32_t)length, 16);
    writeBits(w, (uint16_t)~(uint16_t)length, 16);
}
static void writeTokens(bw_t *w, const uint32_t *toks, uint32_t n, const uint32_t *le, const uint32_t *oe) {
    if (n == 0) return;
    int deferEOB = 0;
    if (toks[n - 1] == END_BLOCK) { n--; deferEOB = 1; }
    for (uint32_t k = 0; k < n; k++) {
        uint32_t t = toks[k];
        if (t < 256) { writeCode(w, le[t]); continue; }
        uint32_t length = (t >> LENGTH_SHIFT) & 0xff;
        uint32_t lc = lengthCode(length) & 31;
        writeCode(w, le[257 + lc]);
        if (lc >= 8) writeBits(w, length - lengthBase[lc], lengthExtraBits[lc]);
        uint32_t offset = t & ((1u << LENGTH_SHIFT) - 1);
        uint32_t oc = (offset >> 16) & 31;
        writeCode(w, oe[oc]);
        if (oc >= 4) writeBits(w, (offset - offsetBase[oc]) & 0xffff, (unsigned)offsetExtraBits[oc]);
    }
    if (deferEOB) writeCode(w, le[END_BLOCK]);
}
static void bw_indexTokens(bw_t *w, const tokens_t *t, int *numLiterals, int *numOffsets) {   /* :784-815, alwaysEOB */
    memcpy(w->literalFreq, t->litHist, 512);
    memcpy(w->literalFreq + 256, t->extraHist, 64);
    memcpy(w->offsetFreq, t->offHist, 64);
    *numLiterals = *numOffsets = 0;
    if (t->n == 0) return;
    w->literalFreq[END_BLOCK] = 1;
    int nl = 289;
    while (w->literalFreq[nl - 1] == 0) nl--;
    int no = 32;
    while (no > 0 && w->offsetFreq[no - 1] == 0) no--;
    if (no == 0) { w->offsetFreq[0] = 1; no = 1; }
    *numLiterals = nl; *numOffsets = no;
}
static void bw_generate(bw_t *w) {
    henc_generate(w->literalEncoding, w->literalFreq, LITERAL_COUNT, 15);
    henc_generate(&w->offsetEncoding, w->offsetFreq, OFFSET_CODE_COUNT, 15);
}
static int canReuse(const bw_t *w, const tokens_t *t) {
    for (int i = 0; i < OFFSET_CODE_COUNT; i++) if (t->offHist[i] && w->offsetEncoding.codes[i] == 0) return 0;
    for (int i = 0; i < LITERAL_COUNT - 256; i++) if (t->extraHist[i] && w->literalEncoding->codes[256 + i] == 0) return 0;
    for (int i = 0; i < 256; i++) if (t->litHist[i] && w->literalEncoding->codes[i] == 0) return 0;
    return 1;
}
static void stored_block(bw_t *w, const uint8_t *in, size_t n, int eof) {
    writeStoredHeader(w, (int)n, eof);
    writeBytes(w, in, n);
}

static void writeBlockDynamic(bw_t *w, tokens_t *tokens, int eof, const uint8_t *input, size_t inlen, int sync) {
    sync = sync || eof;
    if (sync) tok_eob(tokens);
    if ((w->lastHuffMan || eof) && w->lastHeader > 0) {
        writeCode(w, w->literalEncoding->codes[END_BLOCK]);
        w->lastHeader = 0; w->lastHuffMan = 0;
    }
    if (w->lastHeader > 0 && !canReuse(w, tokens)) { writeCode(w, w->literalEncoding->codes[END_BLOCK]); w->lastHeader = 0; }
    int numLiterals, numOffsets;
    bw_indexTokens(w, tokens, &numLiterals, &numOffsets);
    int extraBits = 0, storable;
    int ssize = storedSize(input, inlen, &storable);
    if (storable || w->lastHeader > 0) extraBits = extraBitSize(w);
    int size = 0;
    if (w->lastHeader > 0) {
        int newSize = w->lastHeader + estimatedBits(tokens);
        newSize += hlen(w->literalEncoding->codes[END_BLOCK]) + (newSize >> w->logNewTablePenalty);
        int reuseSize = dynamicReuseSize(w, w->literalEncoding, &w->offsetEncoding) + extraBits;
        if (newSize < reuseSize) {
            writeCode(w, w->literalEncoding->codes[END_BLOCK]);
            size = newSize;
            w->lastHeader = 0;
        } else {
            size = reuseSize;
        }
        if (tokens->n < MAX_PREDEFINED_TOKENS) {
            int preSize = fixedSize(w, extraBits) + 7;
            if (preSize < size) {
                if (storable && ssize <= size) { g_paths[DP_DYN_STORED]++; stored_block(w, input, inlen, eof); return; }
                g_paths[DP_DYN_FIXED]++;
                writeFixedHeader(w, eof);
                if (!sync) tok_eob(tokens);
                writeTokens(w, tokens->tokens, tokens->n, fixedLit.codes, fixedOff.codes);
                return;
            }
        }
        if (storable && ssize <= size) { g_paths[DP_DYN_STORED]++; stored_block(w, input, inlen, eof); return; }
    }
    if (w->lastHeader == 0) {
        w->literalFreq[END_BLOCK] = 1;
        bw_generate(w);
        generateCodegen(w, numLiterals, numOffsets, w->literalEncoding, &w->offsetEncoding);
        henc_generate(&w->codegenEncoding, w->codegenFreq, CODEGEN_COUNT, 7);
        int numCodegens = codegens(w);
        size = dynamicSize(w, w->literalEncoding, &w->offsetEncoding, extraBits);
        if (tokens->n < MAX_PREDEFINED_TOKENS) {
            int preSize = fixedSize(w, extraBits);
            if (preSize <= size) {
                if (storable && ssize <= preSize) { g_paths[DP_DYN_STORED]++; stored_block(w, input, inlen, eof); return; }
                g_paths[DP_DYN_FIXED]++;
                writeFixedHeader(w, eof);
                if (!sync) tok_eob(tokens);
                writeTokens(w, tokens->tokens, tokens->n, fixedLit.codes, fixedOff.codes);
                return;
            }
        }
        if (storable && ssize <= size) { g_paths[DP_DYN_STORED]++; stored_block(w, input, inlen, eof); return; }
        g_paths[DP_DYN_NEW]++;
        writeDynamicHeader(w, numLiterals, numOffsets, numCodegens, eof);
        if (!sync) w->lastHeader = headerSize(w);
        w->lastHuffMan = 0;
    } else {
        g_paths[DP_DYN_REUSE]++;
    }
    if (sync) w->lastHeader = 0;
    writeTokens(w, tokens->tokens, tokens->n, w->literalEncoding->codes, w->offsetEncoding.codes);
}

static void writeBlockHuff(bw_t *w, int eof, const uint8_t *input, size_t inlen, int sync) {
    memset(w->literalFreq, 0, sizeof w->literalFreq);
    if (!w->lastHuffMan) memset(w->offsetFreq, 0, sizeof w->offsetFreq);
    const int numLiterals = END_BLOCK + 1, numOffsets = 1;
    const int guessHeaderSizeBits = 70 * 8;
    for (size_t i = 0; i < inlen; i++) w->literalFreq[input[i]]++;
    int storable;
    int ssize = storedSize(input, inlen, &storable);
    if (storable && inlen > 1024) {
        double abs = 0, avg = (double)inlen / 256, max = (double)(inlen * 2);
        for (int i = 0; i < 256; i++) {
            double diff = (double)w->literalFreq[i] - avg;
            abs += diff * diff;
            if (abs > max) break;
        }
        if (abs < max) { g_paths[DP_HUFF_STORED_TEST]++; stored_block(w, input, inlen, eof); return; }
    }
    w->literalFreq[END_BLOCK] = 1;
    henc_generate(w->tmpLitEncoding, w->literalFreq, numLiterals, 15);
    int estBits = henc_canReuseBits(w->tmpLitEncoding, w->literalFreq, numLiterals);
    if (estBits < 0x7fffffff) {
        estBits += w->lastHeader;
        if (w->lastHeader == 0) estBits += guessHeaderSizeBits;
        estBits += estBits >> w->logNewTablePenalty;
    }
    if (storable && ssize <= estBits) { g_paths[DP_HUFF_STORED_EST]++; stored_block(w, input, inlen, eof); return; }
    if (w->lastHeader > 0) {
        int reuseSize = henc_canReuseBits(w->literalEncoding, w->literalFreq, 256);
        if (estBits < reuseSize) { writeCode(w, w->literalEncoding->codes[END_BLOCK]); w->lastHeader = 0; }
    }
    if (w->lastHeader == 0) {
        g_paths[DP_HUFF_NEW]++;
        henc *t = w->literalEncoding; w->literalEncoding = w->tmpLitEncoding; w->tmpLitEncoding = t;
        generateCodegen(w, numLiterals, numOffsets, w->literalEncoding, &huffOffset);
        henc_generate(&w->codegenEncoding, w->codegenFreq, CODEGEN_COUNT, 7);
        writeDynamicHeader(w, numLiterals, numOffsets, codegens(w), eof);
        w->lastHuffMan = 1;
        w->lastHeader = headerSize(w);
    } else {
        g_paths[DP_HUFF_REUSE]++;
    }
    for (size_t i = 0; i < inlen; i++) writeCode(w, w->literalEncoding->codes[input[i]]);
    if (eof || sync) { writeCode(w, w->literalEncoding->codes[END_BLOCK]); w->lastHeader = 0; w->lastHuffMan = 0; }
}

/* ---- statelessEnc (stateless.go:176-325) */
static uint32_t hashSL(uint32_t u) { return (u * 0x1e35a7bdu) >> (32 - 13); }
static uint32_t ld32(const uint8_t *b, int i) { uint32_t v; memcpy(&v, b + i, 4); return v; }
static uint64_t ld64(const uint8_t *b, int i) { uint64_t v; memcpy(&v, b + i, 8); return v; }
static int matchLen(const uint8_t *a, const uint8_t *b, int n) { int k = 0; while (k < n && a[k] == b[k]) k++; return k; }

static void statelessEnc(tokens_t *dst, const uint8_t *src, int len, int startAt) {
    int16_t table[1 << 13];
    memset(table, 0, sizeof table);
    if (len - startAt < 13) { dst->n = 0; return; }
    if (startAt > 0) {
        uint32_t cv = ld32(src, 0);
        for (int i = 0; i < startAt; i++) { table[hashSL(cv)] = (int16_t)i; cv = (cv >> 8) | (uint32_t)src[i + 4] << 24; }
    }
    int s = startAt + 1, nextEmit = startAt, sLimit = len - 11;
    uint32_t cv = ld32(src, s);
    for (;;) {
        int nextS = s, candidate;
        for (;;) {
            uint32_t nextHash = hashSL(cv);
            candidate = table[nextHash];
            nextS = s + 2 + ((s - nextEmit) >> 5);
            if (nextS > sLimit) goto emitRemainder;   /* int16 wrap-around of nextS also lands here (nextS <= 0) */
            uint64_t now = ld64(src, nextS);
            table[nextHash] = (int16_t)s;
            nextHash = hashSL((uint32_t)now);
            if (cv == ld32(src, candidate)) { table[nextHash] = (int16_t)nextS; break; }
            cv = (uint32_t)now;
            s = nextS;
            nextS++;
            candidate = table[nextHash];
            now >>= 8;
            table[nextHash] = (int16_t)s;
            if (cv == ld32(src, candidate)) { table[nextHash] = (int16_t)nextS; break; }
            cv = (uint32_t)now;
            s = nextS;
        }
        for (;;) {
            int t = candidate;
            int l = matchLen(src + s + 4, src + t + 4, len - s - 4) + 4;
            while (t > 0 && s > nextEmit && src[t - 1] == src[s - 1]) { s--; t--; l++; }
            for (int i = nextEmit; i < s; i++) tok_lit(dst, src[i]);
            tok_match_long(dst, l, (uint32_t)(s - t - 1));
            s += l;
            nextEmit = s;
            if (nextS >= s) s = nextS + 1;
            if (s >= sLimit) goto emitRemainder;
            uint64_t x = ld64(src, s - 2);
            int o = s - 2;
            table[hashSL((uint32_t)x)] = (int16_t)o;
            x >>= 16;
            uint32_t currHash = hashSL((uint32_t)x);
            candidate = table[currHash];
            table[currHash] = (int16_t)(o + 2);
            if ((uint32_t)x != ld32(src, candidate)) { cv = (uint32_t)(x >> 8); s++; break; }
        }
    }
emitRemainder:
    if (nextEmit < len) {
        if (dst->n == 0) return;
        for (int i = nextEmit; i < len; i++) tok_lit(dst, src[i]);
    }
}

/* StatelessDeflate :76-162 into w */
static void stateless(bw_t *w, const uint8_t *in, size_t n, int eof, const uint8_t *dict, size_t dlen) {
    w->bits = 0; w->nbits = 0; w->lastHeader = 0; w->lastHuffMan = 0;
    if (eof && n == 0) { writeStoredHeader(w, 0, 1); bw_flush(w); return; }
    if (dlen > MAX_STATELESS_DICT) { dict += dlen - MAX_STATELESS_DICT; dlen = MAX_STATELESS_DICT; }
    tokens_t dst;
    dst.tokens = malloc((MAX_STORE_BLOCK + 1) * sizeof(uint32_t));
    tok_reset(&dst);
    uint8_t *buf = malloc(MAX_STATELESS_BLOCK + 16);
    const uint8_t *inDict = NULL;
    while (n > 0) {
        size_t todo = n;
        if (inDict) { if (todo > MAX_STATELESS_BLOCK - MAX_STATELESS_DICT) todo = MAX_STATELESS_BLOCK - MAX_STATELESS_DICT; }
        else if (todo > MAX_STATELESS_BLOCK - dlen) todo = MAX_STATELESS_BLOCK - dlen;
        const uint8_t *blk = in;
        in += todo; n -= todo;
        if (inDict) {
            memcpy(buf, inDict, MAX_STATELESS_DICT + todo);
            statelessEnc(&dst, buf, (int)(MAX_STATELESS_DICT + todo), MAX_STATELESS_DICT);
        } else {
            if (dlen) memcpy(buf, dict, dlen);
            memcpy(buf + dlen, blk, todo);
            statelessEnc(&dst, buf, (int)(dlen + todo), (int)dlen);
        }
        int isEof = eof && n == 0;
        if (dst.n == 0) {
            g_paths[DP_STORED_EMPTY_TOKENS]++;
            stored_block(w, blk, todo, isEof);
        } else if ((int)dst.n > (int)todo - (int)(todo >> 4)) {
            writeBlockHuff(w, isEof, blk, todo, n == 0);
        } else {
            writeBlockDynamic(w, &dst, isEof, blk, todo, n == 0);
        }
        if (n > 0) { inDict = blk + todo - MAX_STATELESS_DICT; dict = NULL; dlen = 0; tok_reset(&dst); }
    }
    if (!eof) writeStoredHeader(w, 0, 0);
    bw_flush(w);
    free(buf); free(dst.tokens);
}

/* out gets StatelessDeflate(out, in, eof, dict); returns its bytes or ORC_ERR_DST_SMALL */
ORC_API int64_t orc_deflate_stateless(const uint8_t *in, size_t n, int eof, const uint8_t *dict, size_t dlen, uint8_t *out,
                                      size_t cap) {
    bw_t *w = malloc(sizeof *w);
    bw_init(w, out, cap);
    stateless(w, in, n, eof, dict, dlen);
    int64_t r = w->overflow ? ORC_ERR_DST_SMALL : (int64_t)w->n;
    free(w);
    return r;
}

static uint32_t crc32_upd(uint32_t crc, const uint8_t *p, size_t n) {
    crc = ~crc;
    for (size_t i = 0; i < n; i++) {
        crc ^= p[i];
        for (int k = 0; k < 8; k++) crc = (crc & 1) ? (crc >> 1) ^ 0xedb88320u : crc >> 1;
    }
    return ~crc;
}

/* one gzip member of gzip.NewWriterLevel(w, StatelessCompression): hdr (the header bytes Write emits first), then
 * Write(in) = StatelessDeflate(in, false), then Close = StatelessDeflate(nil, true), CRC-32 and ISIZE */
ORC_API int64_t orc_deflate_gzip(const uint8_t *hdr, size_t hlen, const uint8_t *in, size_t n, uint8_t *out, size_t cap) {
    bw_t *w = malloc(sizeof *w);
    bw_init(w, out, cap);
    writeBytes(w, hdr, hlen);
    stateless(w, in, n, 0, NULL, 0);
    stateless(w, NULL, 0, 1, NULL, 0);
    uint32_t crc = crc32_upd(0, in, n), isz = (uint32_t)n;
    for (int k = 0; k < 4; k++) bw_byte(w, (uint8_t)(crc >> (8 * k)));
    for (int k = 0; k < 4; k++) bw_byte(w, (uint8_t)(isz >> (8 * k)));
    int64_t r = w->overflow ? ORC_ERR_DST_SMALL : (int64_t)w->n;
    free(w);
    return r;
}

/* huffman_bit_writer_test.go testBlockHuff: writeBlockHuff(false, in, false) then flush, with the given penalty */
ORC_API int64_t orc_deflate_block_huff(const uint8_t *in, size_t n, unsigned penalty, uint8_t *out, size_t cap) {
    bw_t *w = malloc(sizeof *w);
    bw_init(w, out, cap);
    w->logNewTablePenalty = penalty;
    writeBlockHuff(w, 0, in, n, 0);
    bw_flush(w);
    int64_t r = w->overflow ? ORC_ERR_DST_SMALL : (int64_t)w->n;
    free(w);
    return r;
}

/* testBlock "dyn" / "sync": indexTokens(toks) then writeBlockDynamic(&tok, false, input, sync) and flush; input may be
 * NULL (the -noinput expectations) */
ORC_API int64_t orc_deflate_block_dynamic(const uint32_t *toks, size_t ntok, const uint8_t *in, size_t n, int sync,
                                          uint8_t *out, size_t cap) {
    bw_t *w = malloc(sizeof *w);
    bw_init(w, out, cap);
    tokens_t t;
    t.tokens = malloc((ntok + 2) * sizeof(uint32_t));
    tok_reset(&t);
    for (size_t i = 0; i < ntok; i++) {
        uint32_t tok = toks[i];
        if (tok < MATCH_TYPE) tok_lit(&t, (uint8_t)tok);
        else tok_match(&t, (tok >> LENGTH_SHIFT) & 0xff, tok & 0xffff);
    }
    writeBlockDynamic(w, &t, 0, in, n, sync);
    bw_flush(w);
    int64_t r = w->overflow ? ORC_ERR_DST_SMALL : (int64_t)w->n;
    free(t.tokens); free(w);
    return r;
}

/* the decision-path counters (DP_* order), and their reset */
ORC_API void orc_deflate_paths(int64_t *out) { memcpy(out, g_paths, sizeof g_paths); }
ORC_API void orc_deflate_paths_reset(void) { memset(g_paths, 0, sizeof g_paths); }
