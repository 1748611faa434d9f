// b2c_deflate.cuh -- flate.StatelessDeflate on the device (flate/stateless.go), raw and inside gzip members written as
// gzip.NewWriterLevel(w, StatelessCompression) writes them (gzip/gzip.go:171-290); byte-identical to the reference.
//
// StatelessDeflate cuts its input at fixed places: block 0 is the first 32767 - len(dict) bytes (dict: the last 8 KiB
// of the one given), every later block the next 24575 bytes with the 8 KiB before it as history.  Each block is parsed
// by statelessEnc with a fresh table, so every block of every input is parsed at once:
//   parse:  one warp per block (block slot = input * max_blocks + k).  Lane 0 runs statelessEnc exactly, with its
//           2^13-entry int16 table in shared memory; the tokens and the three histograms go to the block's slot.
//   encode: one lane per input walks its blocks in order through the reference's huffmanBitWriter (writeBlockDynamic,
//           writeBlockHuff, stored blocks, the table reuse decided by lastHeader / lastHuffMan) and writes the bytes.
//           Its state lives in global memory, so an input whose blocks span several scratch passes carries it across.
//   crc:    one warp per input: the CRC-32 of the input (the inflate kernels' warp CRC, folded onto the seed) and, for
//           gzip, the trailer.
// Floating point: EstimatedBits (float32) and the Huffman-only test (float64) feed byte-changing decisions, so they are
// written with explicitly rounded intrinsics in the reference's order; nothing is contracted into an FMA.
#pragma once
#include "b2c_common.cuh"
#include "b2c_inflate.cuh"

namespace b2c {

constexpr uint32_t DFL_BLOCK0 = 32767, DFL_STEP = 24575, DFL_DICT = 8192;
constexpr uint32_t DFL_SLOT_TOKENS = 32768;            // tokens of one block, EOB included (a block is at most 32767 bytes)
constexpr int DFL_LIT = 286, DFL_OFF = 30, DFL_EOB = 256, DFL_CG = 19;
constexpr int DFL_FMT_RAW = 0, DFL_FMT_GZIP = 2;      // and DFL_FMT_ZLIB (BestSpeed only)

struct DflSlot {                                       // one parsed block
    uint32_t n, pad[3];
    uint16_t extraHist[32], offHist[32], litHist[256];
};
struct DflHenc { uint32_t codes[320]; int32_t bitCount[17]; };
struct DflState {                                      // the huffmanBitWriter of one input, kept across passes
    uint64_t bits, n;
    uint32_t nbits, overflow;
    int32_t lastHeader, lastHuffMan, litSel, pad;
    DflHenc lit[2], off, cg;
    uint16_t literalFreq[289], offsetFreq[32], codegenFreq[DFL_CG];
    uint8_t codegen[DFL_LIT + DFL_OFF + 1];
};

struct DflParams {
    const uint8_t *src_base; size_t src_stride; const uint64_t *src_offsets; const uint32_t *src_sizes;
    const uint8_t *dict_base; const uint64_t *dict_offsets; const uint32_t *dict_sizes;   // dict_sizes null: no dicts
    const uint8_t *eof;                                // null: every input ends its stream
    uint8_t *dst_base; size_t dst_stride; const uint64_t *dst_offsets; uint32_t dst_cap; const uint32_t *dst_caps;
    int64_t *out_sizes;
    const uint32_t *crc_in; uint32_t *crc_out;
    const uint8_t *hdr; uint32_t hlen;
    int format;
    uint32_t max_blocks;
    uint64_t g0, g1;                                   // the block slots of this pass
    DflSlot *slots; uint32_t *tokens;                  // per slot of the pass
    DflState *state;                                   // per input
};

B2C_DEV const uint8_t *dfl_src(const DflParams &P, uint32_t i) {
    return P.src_base + (P.src_offsets ? P.src_offsets[i] : (uint64_t)i * P.src_stride);
}
B2C_DEV uint8_t *dfl_dst(const DflParams &P, uint32_t i) {
    return P.dst_base + (P.dst_offsets ? P.dst_offsets[i] : (uint64_t)i * P.dst_stride);
}
B2C_DEV uint32_t dfl_cap(const DflParams &P, uint32_t i) { return P.dst_caps ? P.dst_caps[i] : P.dst_cap; }
B2C_DEV uint32_t dfl_dict_len(const DflParams &P, uint32_t i) {
    const uint32_t d = P.dict_sizes ? P.dict_sizes[i] : 0;
    return d > DFL_DICT ? DFL_DICT : d;
}
B2C_DEV const uint8_t *dfl_dict(const DflParams &P, uint32_t i) {   // the last dfl_dict_len bytes of input i's dict
    return P.dict_base + P.dict_offsets[i] + (P.dict_sizes[i] - dfl_dict_len(P, i));
}
// blocks of an input of n bytes whose dict counts d bytes (0 for an empty input)
__host__ __device__ inline uint32_t dfl_blocks(uint64_t n, uint32_t d) {
    const uint64_t b0 = DFL_BLOCK0 - d;
    return n == 0 ? 0 : (uint32_t)(1 + (n > b0 ? (n - b0 + DFL_STEP - 1) / DFL_STEP : 0));
}

// ---- parse: statelessEnc (stateless.go:176-325) on lane 0 of a warp
// The block's source is hist[0, hl) followed by in[0, len): the dict (block 0) or the 8 KiB before the block.
struct DflSrc {
    const uint8_t *hist, *in; int hl;
    B2C_DEV uint8_t at(int i) const { return i < hl ? hist[i] : in[i - hl]; }
    B2C_DEV uint32_t ld32(int i) const {
        return (uint32_t)at(i) | (uint32_t)at(i + 1) << 8 | (uint32_t)at(i + 2) << 16 | (uint32_t)at(i + 3) << 24;
    }
    B2C_DEV uint64_t ld64(int i) const { return (uint64_t)ld32(i) | (uint64_t)ld32(i + 4) << 32; }
};
__constant__ uint8_t dfl_lbase[32] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 10, 12, 14, 16, 20, 24, 28, 32, 40, 48, 56, 64, 80, 96,
                                      112, 128, 160, 192, 224, 255};
__constant__ uint8_t dfl_lextra[32] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
__constant__ int8_t dfl_oextra[32] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11,
                                      12, 12, 13, 13, 14, 14};
__constant__ uint32_t dfl_obase[32] = {0x0000, 0x0001, 0x0002, 0x0003, 0x0004, 0x0006, 0x0008, 0x000c, 0x0010, 0x0018,
                                       0x0020, 0x0030, 0x0040, 0x0060, 0x0080, 0x00c0, 0x0100, 0x0180, 0x0200, 0x0300,
                                       0x0400, 0x0600, 0x0800, 0x0c00, 0x1000, 0x1800, 0x2000, 0x3000, 0x4000, 0x6000};
__constant__ uint8_t dfl_cgorder[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

B2C_DEV uint32_t dfl_lcode(uint32_t len) {             // lengthCodes (token.go:30-57)
    uint32_t c = 0;
    while (c < 28 && dfl_lbase[c + 1] <= len) c++;
    return c;
}
B2C_DEV uint32_t dfl_ocode(uint32_t off) {             // offsetCode (token.go:365-379)
    if (off < 4) return off;
    const uint32_t hb = highbit32(off);
    return 2 * hb + ((off >> (hb - 1)) & 1);
}
B2C_DEV uint32_t dfl_hash(uint32_t u) { return (u * 0x1e35a7bdu) >> (32 - 13); }

struct DflTok {
    DflSlot *s; uint32_t *t;
    B2C_DEV void lit(uint8_t v) { t[s->n++] = v; s->litHist[v]++; }
    B2C_DEV void match_long(int32_t xlength, uint32_t xoffset) {      // AddMatchLong (token.go:284-309)
        const uint32_t oc = dfl_ocode(xoffset);
        xoffset |= oc << 16;
        while (xlength > 0) {
            int32_t xl = xlength;
            if (xl > 258) xl = xl > 258 + 3 ? 258 : 258 - 3;
            xlength -= xl;
            xl -= 3;
            s->extraHist[dfl_lcode((uint32_t)xl) + 1]++;
            s->offHist[oc & 31]++;
            t[s->n++] = (1u << 30) | (uint32_t)xl << 22 | xoffset;
        }
    }
};

B2C_DEV void dfl_parse(const DflSrc &src, int len, int startAt, DflTok &dst, int16_t *table) {
    if (len - startAt < 13) return;
    if (startAt > 0) {
        uint32_t cv = src.ld32(0);
        for (int i = 0; i < startAt; i++) { table[dfl_hash(cv)] = (int16_t)i; cv = (cv >> 8) | (uint32_t)src.at(i + 4) << 24; }
    }
    int s = startAt + 1, nextEmit = startAt;
    const int sLimit = len - 11;
    uint32_t cv = src.ld32(s);
    for (;;) {
        int nextS = s, candidate;
        for (;;) {
            uint32_t nextHash = dfl_hash(cv);
            candidate = table[nextHash];
            nextS = s + 2 + ((s - nextEmit) >> 5);
            if (nextS > sLimit) goto emitRemainder;   // the reference's int16 wrap-around (nextS <= 0) also lands here
            uint64_t now = src.ld64(nextS);
            table[nextHash] = (int16_t)s;
            nextHash = dfl_hash((uint32_t)now);
            if (cv == src.ld32(candidate)) { table[nextHash] = (int16_t)nextS; break; }
            cv = (uint32_t)now;
            s = nextS;
            nextS++;
            candidate = table[nextHash];
            now >>= 8;
            table[nextHash] = (int16_t)s;
            if (cv == src.ld32(candidate)) { table[nextHash] = (int16_t)nextS; break; }
            cv = (uint32_t)now;
            s = nextS;
        }
        for (;;) {
            int t = candidate;
            int l = 4;
            while (s + l < len && src.at(s + l) == src.at(t + l)) l++;
            while (t > 0 && s > nextEmit && src.at(t - 1) == src.at(s - 1)) { s--; t--; l++; }
            for (int i = nextEmit; i < s; i++) dst.lit(src.at(i));
            dst.match_long(l, (uint32_t)(s - t - 1));
            s += l;
            nextEmit = s;
            if (nextS >= s) s = nextS + 1;
            if (s >= sLimit) goto emitRemainder;
            uint64_t x = src.ld64(s - 2);
            const int o = s - 2;
            table[dfl_hash((uint32_t)x)] = (int16_t)o;
            x >>= 16;
            const uint32_t currHash = dfl_hash((uint32_t)x);
            candidate = table[currHash];
            table[currHash] = (int16_t)(o + 2);
            if ((uint32_t)x != src.ld32(candidate)) { cv = (uint32_t)(x >> 8); s++; break; }
        }
    }
emitRemainder:
    if (nextEmit < len && dst.s->n != 0)
        for (int i = nextEmit; i < len; i++) dst.lit(src.at(i));
}

// An input larger than src_stride (the bound the slot grid was sized from) is refused: B2C_ERR_ARG, nothing read
constexpr int64_t DFL_ERR_ARG = -102;
B2C_DEV bool dfl_too_big(const DflParams &P, uint32_t i) { return P.src_stride && P.src_sizes[i] > P.src_stride; }

// the block of slot g: its input, index, source and length
struct DflBlock { uint32_t input, k, nblocks; uint64_t start; uint32_t len; int hl; };
B2C_DEV bool dfl_block(const DflParams &P, uint64_t g, uint32_t nchunks, DflBlock &b) {
    b.input = (uint32_t)(g / P.max_blocks); b.k = (uint32_t)(g % P.max_blocks);
    if (b.input >= nchunks || dfl_too_big(P, b.input)) return false;
    const uint32_t n = P.src_sizes[b.input], d = dfl_dict_len(P, b.input);
    b.nblocks = dfl_blocks(n, d);
    if (b.k >= b.nblocks) return false;
    const uint64_t b0 = DFL_BLOCK0 - d;
    b.start = b.k == 0 ? 0 : b0 + (uint64_t)(b.k - 1) * DFL_STEP;
    const uint64_t want = b.k == 0 ? b0 : DFL_STEP;
    b.len = (uint32_t)(n - b.start < want ? n - b.start : want);
    b.hl = b.k == 0 ? (int)d : (int)DFL_DICT;
    return true;
}

B2C_DEV void dfl_parse_warp(const DflParams &P, uint64_t g, uint32_t nchunks, int16_t *table, unsigned lane) {
    DflBlock b;
    if (!dfl_block(P, g, nchunks, b)) return;
    DflSlot *slot = P.slots + (g - P.g0);
    for (uint32_t i = lane; i < sizeof(DflSlot) / 4; i += 32) reinterpret_cast<uint32_t *>(slot)[i] = 0;
    for (uint32_t i = lane; i < (1u << 13) / 2; i += 32) reinterpret_cast<uint32_t *>(table)[i] = 0;
    __syncwarp();
    if (lane == 0) {
        const uint8_t *in = dfl_src(P, b.input);
        DflSrc src{b.k == 0 ? (b.hl ? dfl_dict(P, b.input) : in) : in + b.start - DFL_DICT, in + b.start, b.hl};
        DflTok tok{slot, P.tokens + (g - P.g0) * DFL_SLOT_TOKENS};
        dfl_parse(src, b.hl + (int)b.len, b.hl, tok, table);
    }
}

// ---- encode: the huffmanBitWriter (huffman_bit_writer.go) of one input on one lane
B2C_DEV uint16_t dfl_rev(uint16_t number, uint32_t bitLength) {
    return (uint16_t)(__brev((uint32_t)(uint16_t)(number << ((16 - bitLength) & 15))) >> 16);
}
B2C_DEV uint32_t dfl_hcode(uint16_t code, uint32_t len) { return len | (uint32_t)code << 8; }
B2C_DEV uint32_t dfl_fixed_lit(uint32_t ch) {
    uint32_t bits, size;
    if (ch < 144) { bits = ch + 48; size = 8; }
    else if (ch < 256) { bits = ch + 400 - 144; size = 9; }
    else if (ch < 280) { bits = ch - 256; size = 7; }
    else { bits = ch + 192 - 280; size = 8; }
    return dfl_hcode(dfl_rev((uint16_t)bits, size), size);
}
B2C_DEV uint32_t dfl_fixed_off(uint32_t ch) { return dfl_hcode(dfl_rev((uint16_t)ch, 5), 5); }

B2C_DEV int dfl_bitlen(const uint32_t *codes, const uint16_t *freq, int n) {
    int total = 0;
    for (int i = 0; i < n; i++) if (freq[i]) total += freq[i] * (int)(codes[i] & 0xff);
    return total;
}
B2C_DEV int dfl_reuse_bits(const uint32_t *codes, const uint16_t *freq, int n) {    // canReuseBits
    int total = 0;
    for (int i = 0; i < n; i++)
        if (freq[i]) {
            if (codes[i] == 0) return 0x7fffffff;
            total += freq[i] * (int)(codes[i] & 0xff);
        }
    return total;
}

// huffmanEncoder.generate (huffman_code.go:339-371) with bitCounts and assignEncodingAndSize.  Literals are distinct,
// so ordering by (freq, literal) and by literal with any sort gives the reference's order.
B2C_DEV void dfl_generate(DflHenc *h, const uint16_t *freq, int nfreq, int32_t maxBits) {
    uint32_t list[DFL_LIT + 1];                        // freq << 16 | literal
    int count = 0;
    for (int i = 0; i < nfreq; i++) {
        if (freq[i]) list[count++] = (uint32_t)freq[i] << 16 | (uint32_t)i;
        else h->codes[i] = 0;
    }
    if (count <= 2) {
        for (int i = 0; i < count; i++) h->codes[list[i] & 0xffff] = dfl_hcode((uint16_t)i, 1);
        return;
    }
    for (int i = 1; i < count; i++) {
        const uint32_t v = list[i];
        int j = i;
        for (; j > 0 && list[j - 1] > v; j--) list[j] = list[j - 1];
        list[j] = v;
    }
    const int32_t n = count;
    if (maxBits > n - 1) maxBits = n - 1;
    int32_t lastFreq[16], nextCharFreq[16], nextPairFreq[16], needed[16];
    int32_t leafCounts[16][16];
    for (int i = 0; i < 16; i++) {
        lastFreq[i] = nextCharFreq[i] = nextPairFreq[i] = needed[i] = 0;
        for (int j = 0; j < 16; j++) leafCounts[i][j] = 0;
    }
    auto fq = [&](int k) -> int32_t { return k < n ? (int32_t)(list[k] >> 16) : 0x7fffffff; };
    const int32_t l2f = fq(2), l1f = fq(1), l0f = fq(0) + fq(1);
    for (int32_t level = 1; level <= maxBits; level++) {
        lastFreq[level] = l1f; nextCharFreq[level] = l2f; nextPairFreq[level] = l0f; needed[level] = 0;
        leafCounts[level][level] = 2;
        if (level == 1) nextPairFreq[level] = 0x7fffffff;
    }
    needed[maxBits] = 2 * n - 4;
    uint32_t level = (uint32_t)maxBits;
    while (level < 16) {
        if (nextPairFreq[level] == 0x7fffffff && nextCharFreq[level] == 0x7fffffff) {
            needed[level] = 0;
            if (level + 1 < 16) nextPairFreq[level + 1] = 0x7fffffff;
            level++;
            continue;
        }
        const int32_t prevFreq = lastFreq[level];
        if (nextCharFreq[level] < nextPairFreq[level]) {
            const int32_t nn = leafCounts[level][level] + 1;
            lastFreq[level] = nextCharFreq[level];
            leafCounts[level][level] = nn;
            nextCharFreq[level] = fq(nn);              // the sentinel after the list is maxNode: MaxInt32
        } else {
            lastFreq[level] = nextPairFreq[level];
            const int32_t save = leafCounts[level][level];
            for (int j = 0; j < 16; j++) leafCounts[level][j] = leafCounts[level - 1][j];
            leafCounts[level][level] = save;
            needed[level - 1] = 2;
        }
        if (--needed[level] == 0) {
            if ((int32_t)level == maxBits) break;
            nextPairFreq[level + 1] = prevFreq + lastFreq[level];
            level++;
        } else {
            while (needed[level - 1] > 0) level--;
        }
    }
    int32_t bitCount[17];
    bitCount[0] = 0;
    for (int32_t lv = maxBits, bits = 1; lv > 0; lv--, bits++) bitCount[bits] = leafCounts[maxBits][lv] - leafCounts[maxBits][lv - 1];
    uint16_t code = 0;
    int len = count;
    for (int b = 0; b <= maxBits; b++) {
        code <<= 1;
        const int32_t bits = bitCount[b];
        if (b == 0 || bits == 0) continue;
        uint32_t *chunk = list + len - bits;           // sort by literal
        for (int i = 1; i < bits; i++) {
            const uint32_t v = chunk[i];
            int j = i;
            for (; j > 0 && (chunk[j - 1] & 0xffff) > (v & 0xffff); j--) chunk[j] = chunk[j - 1];
            chunk[j] = v;
        }
        for (int i = 0; i < bits; i++) { h->codes[chunk[i] & 0xffff] = dfl_hcode(dfl_rev(code, (uint32_t)b), (uint32_t)b); code++; }
        len -= bits;
    }
}

struct DflWriter {
    DflState *st;
    uint8_t *out; uint64_t cap;
    uint64_t bits, n; uint32_t nbits; bool overflow;
    int lastHeader, lastHuffMan, litSel;

    B2C_DEV DflHenc *lit() { return &st->lit[litSel]; }
    B2C_DEV void byte(uint8_t v) { if (n < cap) out[n] = v; else overflow = true; n++; }
    B2C_DEV void put(uint32_t b, uint32_t nb) {
        bits |= (uint64_t)b << nbits;
        nbits += nb;
        while (nbits >= 8) { byte((uint8_t)bits); bits >>= 8; nbits -= 8; }
    }
    B2C_DEV void code(uint32_t c) { put(c >> 8, c & 0xff); }
    B2C_DEV void flush() {
        if (lastHeader > 0) { code(lit()->codes[DFL_EOB]); lastHeader = 0; }
        if (nbits) { byte((uint8_t)bits); bits = 0; nbits = 0; }
    }
    B2C_DEV void fixed_header(bool eof) {
        if (lastHeader > 0) { code(lit()->codes[DFL_EOB]); lastHeader = 0; }
        put(eof ? 3 : 2, 3);
    }
    B2C_DEV void stored_header(uint32_t length, bool eof) {
        if (lastHeader > 0) { code(lit()->codes[DFL_EOB]); lastHeader = 0; }
        if (length == 0 && eof) { fixed_header(true); put(0, 7); flush(); return; }
        put(eof ? 1 : 0, 3);
        flush();
        put(length, 16);
        put((uint16_t)~(uint16_t)length, 16);
    }
    B2C_DEV void stored(const uint8_t *in, uint32_t len, bool eof) {
        stored_header(len, eof);
        for (uint32_t i = 0; i < len; i++) byte(in[i]);
    }
    B2C_DEV void gen_codegen(int numLiterals, int numOffsets, const uint32_t *litc, const uint32_t *offc) {
        uint16_t *cf = st->codegenFreq;
        uint8_t *cg = st->codegen;
        for (int i = 0; i < DFL_CG; i++) cf[i] = 0;
        for (int i = 0; i < numLiterals; i++) cg[i] = (uint8_t)(litc[i] & 0xff);
        for (int i = 0; i < numOffsets; i++) cg[numLiterals + i] = (uint8_t)(offc[i] & 0xff);
        cg[numLiterals + numOffsets] = 255;
        uint8_t size = cg[0];
        int count = 1, outIndex = 0;
        for (int inIndex = 1; size != 255; inIndex++) {
            const uint8_t nextSize = cg[inIndex];
            if (nextSize == size) { count++; continue; }
            if (size != 0) {
                cg[outIndex++] = size; cf[size]++;
                count--;
                while (count >= 3) {
                    const int k = count < 6 ? count : 6;
                    cg[outIndex++] = 16; cg[outIndex++] = (uint8_t)(k - 3); cf[16]++;
                    count -= k;
                }
            } else {
                while (count >= 11) {
                    const int k = count < 138 ? count : 138;
                    cg[outIndex++] = 18; cg[outIndex++] = (uint8_t)(k - 11); cf[18]++;
                    count -= k;
                }
                if (count >= 3) { cg[outIndex++] = 17; cg[outIndex++] = (uint8_t)(count - 3); cf[17]++; count = 0; }
            }
            count--;
            for (; count >= 0; count--) { cg[outIndex++] = size; cf[size]++; }
            size = nextSize;
            count = 1;
        }
        cg[outIndex] = 255;
    }
    B2C_DEV int codegens() {
        int k = DFL_CG;
        while (k > 4 && st->codegenFreq[dfl_cgorder[k - 1]] == 0) k--;
        return k;
    }
    B2C_DEV int header_size() {
        const uint16_t *cf = st->codegenFreq;
        return 3 + 5 + 5 + 4 + 3 * codegens() + dfl_bitlen(st->cg.codes, cf, DFL_CG) + cf[16] * 2 + cf[17] * 3 + cf[18] * 7;
    }
    B2C_DEV void dynamic_header(int numLiterals, int numOffsets, int numCodegens, bool eof) {
        put(eof ? 5 : 4, 3);
        put((uint32_t)(numLiterals - 257), 5);
        put((uint32_t)(numOffsets - 1), 5);
        put((uint32_t)(numCodegens - 4), 4);
        for (int i = 0; i < numCodegens; i++) put(st->cg.codes[dfl_cgorder[i]] & 0xff, 3);
        for (int i = 0;;) {
            const uint32_t cw = st->codegen[i++];
            if (cw == 255) break;
            code(st->cg.codes[cw]);
            if (cw == 16) put(st->codegen[i++], 2);
            else if (cw == 17) put(st->codegen[i++], 3);
            else if (cw == 18) put(st->codegen[i++], 7);
        }
    }
    // writeTokens with le / oe: the literal / length code and offset code of each token; eob: one EOB at the end
    template <class LE, class OE>
    B2C_DEV void tokens(const uint32_t *toks, uint32_t nt, LE le, OE oe, bool eob) {
        for (uint32_t k = 0; k < nt; k++) {
            const uint32_t t = toks[k];
            if (t < 256) { code(le(t)); continue; }
            const uint32_t length = (t >> 22) & 0xff, lc = dfl_lcode(length);
            code(le(257 + lc));
            if (lc >= 8) put(length - dfl_lbase[lc], dfl_lextra[lc]);
            const uint32_t offset = t & ((1u << 22) - 1), oc = (offset >> 16) & 31;
            code(oe(oc));
            if (oc >= 4) put((offset - dfl_obase[oc]) & 0xffff, (uint32_t)dfl_oextra[oc]);
        }
        if (eob) code(le(DFL_EOB));
    }
};

B2C_DEV float dfl_log2(float val) {                    // mFastLog2 (token.go:212-220)
    int32_t ux = __float_as_int(val);
    float lg = (float)(((ux >> 23) & 255) - 128);
    ux &= -0x7f800001;
    ux += 127 << 23;
    const float uval = __int_as_float(ux);
    lg = __fadd_rn(lg, __fsub_rn(__fmul_rn(__fadd_rn(__fmul_rn(-0.34484843f, uval), 2.02466578f), uval), 0.67487759f));
    return lg;
}
B2C_DEV float dfl_clamp(float v) { return v < 1 ? 1.0f : (v > 15 ? 15.0f : v); }
// EstimatedBits (token.go:225-260) of a slot (nFilled is 0); ntok counts the EOB when the block added one
B2C_DEV int dfl_estimated_bits(const DflSlot *s, uint32_t ntok, const uint16_t *extra) {
    float shannon = 0;
    int bits = 0, nMatches = 0;
    const int total = (int)ntok;
    if (total > 0) {
        const float inv = __fdiv_rn(1.0f, (float)total);
        for (int i = 0; i < 256; i++)
            if (s->litHist[i]) {
                const float n = (float)s->litHist[i];
                shannon = __fadd_rn(shannon, __fmul_rn(dfl_clamp(-dfl_log2(__fmul_rn(n, inv))), n));
            }
        shannon = __fadd_rn(shannon, 15.0f);
        for (int i = 0; i < 29; i++) {
            const uint16_t v = extra[1 + i];
            if (v) {
                const float n = (float)v;
                shannon = __fadd_rn(shannon, __fmul_rn(dfl_clamp(-dfl_log2(__fmul_rn(n, inv))), n));
                bits += dfl_lextra[i] * (int)v;
                nMatches += v;
            }
        }
    }
    if (nMatches > 0) {
        const float inv = __fdiv_rn(1.0f, (float)nMatches);
        for (int i = 0; i < DFL_OFF; i++) {
            const uint16_t v = s->offHist[i];
            if (v) {
                const float n = (float)v;
                shannon = __fadd_rn(shannon, __fmul_rn(dfl_clamp(-dfl_log2(__fmul_rn(n, inv))), n));
                bits += dfl_oextra[i] * (int)v;
            }
        }
    }
    return (int)shannon + bits;
}

// writeBlockDynamic (huffman_bit_writer.go:620-765) for a parsed block.  PEN is the writer's logNewTablePenalty: 0 in the
// stateless path (a pooled writer), 7 at BestSpeed (deflate.go:803-808).
template <int PEN>
B2C_DEV void dfl_block_dynamic(DflWriter &w, const DflSlot *s, const uint32_t *toks, bool eof, const uint8_t *input,
                               uint32_t inlen, bool sync) {
    DflState *st = w.st;
    sync = sync || eof;
    uint32_t ntok = s->n;
    uint16_t extra0 = s->extraHist[0];
    if (sync) { ntok++; extra0++; }                    // AddEOB
    if ((w.lastHuffMan || eof) && w.lastHeader > 0) { w.code(w.lit()->codes[DFL_EOB]); w.lastHeader = 0; w.lastHuffMan = 0; }
    if (w.lastHeader > 0) {                            // canReuse
        bool ok = true;
        for (int i = 0; i < DFL_OFF && ok; i++) ok = !(s->offHist[i] && st->off.codes[i] == 0);
        for (int i = 0; i < DFL_LIT - 256 && ok; i++) ok = !((i ? s->extraHist[i] : extra0) && w.lit()->codes[256 + i] == 0);
        for (int i = 0; i < 256 && ok; i++) ok = !(s->litHist[i] && w.lit()->codes[i] == 0);
        if (!ok) { w.code(w.lit()->codes[DFL_EOB]); w.lastHeader = 0; }
    }
    // indexTokens (alwaysEOB)
    uint16_t *lf = st->literalFreq, *of = st->offsetFreq;
    for (int i = 0; i < 256; i++) lf[i] = s->litHist[i];
    for (int i = 0; i < 32; i++) lf[256 + i] = i ? s->extraHist[i] : extra0;
    lf[288] = 0;
    for (int i = 0; i < 32; i++) of[i] = s->offHist[i];
    lf[DFL_EOB] = 1;
    int numLiterals = 289;
    while (lf[numLiterals - 1] == 0) numLiterals--;
    int numOffsets = 32;
    while (numOffsets > 0 && of[numOffsets - 1] == 0) numOffsets--;
    if (numOffsets == 0) { of[0] = 1; numOffsets = 1; }
    auto extraBitSize = [&]() {
        int total = 0;
        for (int i = 0; i < DFL_LIT - 257; i++) total += lf[257 + i] * dfl_lextra[i];
        for (int i = 0; i < DFL_OFF; i++) total += of[i] * dfl_oextra[i];
        return total;
    };
    auto fixedSize = [&](int extraBits) {
        int t = 3 + extraBits;                         // frequencies past 285 / 29 are zero
        for (int i = 0; i < DFL_LIT; i++) if (lf[i]) t += lf[i] * (int)(dfl_fixed_lit((uint32_t)i) & 0xff);
        for (int i = 0; i < DFL_OFF; i++) t += of[i] * 5;
        return t;
    };
    const bool storable = input != nullptr && inlen <= 65535;
    const int ssize = storable ? (int)(inlen + 5) * 8 : 0;
    const int extraBits = (storable || w.lastHeader > 0) ? extraBitSize() : 0;
    auto fixed_block = [&]() {
        w.fixed_header(eof);
        w.tokens(toks, s->n, [](uint32_t c) { return dfl_fixed_lit(c); }, [](uint32_t c) { return dfl_fixed_off(c); }, true);
    };
    int size = 0;
    if (w.lastHeader > 0) {
        int newSize = w.lastHeader + dfl_estimated_bits(s, ntok, lf + 256);
        newSize += (int)(w.lit()->codes[DFL_EOB] & 0xff) + (newSize >> PEN);
        const int reuseSize = dfl_bitlen(w.lit()->codes, lf, 289) + dfl_bitlen(st->off.codes, of, 32) + extraBits;
        if (newSize < reuseSize) { w.code(w.lit()->codes[DFL_EOB]); size = newSize; w.lastHeader = 0; }
        else size = reuseSize;
        if (ntok < 250 && fixedSize(extraBits) + 7 < size) {
            if (storable && ssize <= size) { w.stored(input, inlen, eof); return; }
            fixed_block();
            return;
        }
        if (storable && ssize <= size) { w.stored(input, inlen, eof); return; }
    }
    if (w.lastHeader == 0) {
        lf[DFL_EOB] = 1;
        dfl_generate(w.lit(), lf, DFL_LIT, 15);
        dfl_generate(&st->off, of, DFL_OFF, 15);
        w.gen_codegen(numLiterals, numOffsets, w.lit()->codes, st->off.codes);
        dfl_generate(&st->cg, st->codegenFreq, DFL_CG, 7);
        const int numCodegens = w.codegens();
        size = w.header_size() + dfl_bitlen(w.lit()->codes, lf, 289) + dfl_bitlen(st->off.codes, of, 32) + extraBits;
        if (ntok < 250) {
            const int preSize = fixedSize(extraBits);
            if (preSize <= size) {
                if (storable && ssize <= preSize) { w.stored(input, inlen, eof); return; }
                fixed_block();
                return;
            }
        }
        if (storable && ssize <= size) { w.stored(input, inlen, eof); return; }
        w.dynamic_header(numLiterals, numOffsets, numCodegens, eof);
        if (!sync) w.lastHeader = w.header_size();
        w.lastHuffMan = 0;
    }
    if (sync) w.lastHeader = 0;
    const uint32_t *lc = w.lit()->codes, *oc = st->off.codes;
    w.tokens(toks, s->n, [lc](uint32_t c) { return lc[c]; }, [oc](uint32_t c) { return oc[c]; }, sync);
}

// writeBlockHuff's quick check for incompressible content (huffman_bit_writer.go:1011-1030), float64 in its order, for
// the HuffmanOnly analysis.  dfl_block_huff keeps its own copy inline: calling this from it reorders the code of the
// kernels that use it.
B2C_DEV bool dfl_huff_incompressible(const uint16_t *lf, uint32_t inlen) {
    double abs = 0;
    const double avg = __ddiv_rn((double)inlen, 256.0), max = (double)(inlen * 2);
    for (int i = 0; i < 256; i++) {
        const double diff = __dsub_rn((double)lf[i], avg);
        abs = __dadd_rn(abs, __dmul_rn(diff, diff));
        if (abs > max) break;
    }
    return abs < max;
}

// writeBlockHuff (huffman_bit_writer.go:987-1174); huffOffset is one code of length 1 for offset 0; PEN as above
template <int PEN>
B2C_DEV void dfl_block_huff(DflWriter &w, bool eof, const uint8_t *input, uint32_t inlen, bool sync) {
    DflState *st = w.st;
    uint16_t *lf = st->literalFreq;
    for (int i = 0; i < 289; i++) lf[i] = 0;
    for (uint32_t i = 0; i < inlen; i++) lf[input[i]]++;
    const bool storable = inlen <= 65535;
    const int ssize = storable ? (int)(inlen + 5) * 8 : 0;
    if (storable && inlen > 1024) {
        double abs = 0;
        const double avg = __ddiv_rn((double)inlen, 256.0), max = (double)(inlen * 2);
        for (int i = 0; i < 256; i++) {
            const double diff = __dsub_rn((double)lf[i], avg);
            abs = __dadd_rn(abs, __dmul_rn(diff, diff));
            if (abs > max) break;
        }
        if (abs < max) { w.stored(input, inlen, eof); return; }
    }
    lf[DFL_EOB] = 1;
    DflHenc *tmp = &st->lit[w.litSel ^ 1];
    dfl_generate(tmp, lf, DFL_EOB + 1, 15);
    int estBits = dfl_reuse_bits(tmp->codes, lf, DFL_EOB + 1);
    if (estBits < 0x7fffffff) {
        estBits += w.lastHeader;
        if (w.lastHeader == 0) estBits += 70 * 8;
        estBits += estBits >> PEN;
    }
    if (storable && ssize <= estBits) { w.stored(input, inlen, eof); return; }
    if (w.lastHeader > 0 && estBits < dfl_reuse_bits(w.lit()->codes, lf, 256)) {
        w.code(w.lit()->codes[DFL_EOB]);
        w.lastHeader = 0;
    }
    if (w.lastHeader == 0) {
        w.litSel ^= 1;
        uint32_t huffOff[1] = {dfl_hcode(0, 1)};
        w.gen_codegen(DFL_EOB + 1, 1, w.lit()->codes, huffOff);
        dfl_generate(&st->cg, st->codegenFreq, DFL_CG, 7);
        w.dynamic_header(DFL_EOB + 1, 1, w.codegens(), eof);
        w.lastHuffMan = 1;
        w.lastHeader = w.header_size();
    }
    const uint32_t *enc = w.lit()->codes;
    for (uint32_t i = 0; i < inlen; i++) w.code(enc[input[i]]);
    if (eof || sync) { w.code(enc[DFL_EOB]); w.lastHeader = 0; w.lastHuffMan = 0; }
}

// One lane: input i's blocks of this pass, in order; the call's end (the empty stored block or the final block's
// flush) after its last block.  Results: out_sizes[i] = deflate bytes so far (the crc kernel adds the gzip trailer).
B2C_DEV void dfl_encode_lane(const DflParams &P, uint32_t i) {
    const uint32_t n = P.src_sizes[i], d = dfl_dict_len(P, i), nb = dfl_blocks(n, d);
    const uint64_t gbase = (uint64_t)i * P.max_blocks;
    if (dfl_too_big(P, i)) {
        if (gbase >= P.g0) P.out_sizes[i] = DFL_ERR_ARG;   // the pass holding the input's first slot
        return;
    }
    const uint32_t k0 = P.g0 > gbase ? (uint32_t)(P.g0 - gbase) : 0;
    const uint64_t kend = P.g1 - gbase;
    const uint32_t k1 = nb < kend ? nb : (uint32_t)kend;
    const bool first = k0 == 0, ends = (nb == 0 && first) || (nb > 0 && k1 == nb && k0 < nb);
    if (!first && k0 >= k1) return;                    // none of this input's blocks is in this pass
    if (first && nb > 0 && k0 >= k1) return;
    const bool eof = P.format == DFL_FMT_GZIP ? false : (P.eof ? P.eof[i] != 0 : true);
    DflState *st = P.state + i;
    DflWriter w;
    w.st = st; w.out = dfl_dst(P, i); w.cap = dfl_cap(P, i);
    if (first) {
        w.bits = 0; w.n = 0; w.nbits = 0; w.overflow = false; w.lastHeader = 0; w.lastHuffMan = 0; w.litSel = 0;
        for (uint32_t k = 0; k < P.hlen; k++) w.byte(P.hdr[k]);
    } else {
        w.bits = st->bits; w.n = st->n; w.nbits = st->nbits; w.overflow = st->overflow != 0;
        w.lastHeader = st->lastHeader; w.lastHuffMan = st->lastHuffMan; w.litSel = st->litSel;
    }
    const uint8_t *in = dfl_src(P, i);
    for (uint32_t k = k0; k < k1 && !w.overflow; k++) {
        DflBlock b;
        dfl_block(P, gbase + k, 0xffffffffu, b);
        const DflSlot *s = P.slots + (gbase + k - P.g0);
        const uint32_t *toks = P.tokens + (gbase + k - P.g0) * DFL_SLOT_TOKENS;
        const bool last = k + 1 == nb, isEof = eof && last;
        const uint8_t *blk = in + b.start;
        if (s->n == 0) w.stored(blk, b.len, isEof);
        else if ((int)s->n > (int)b.len - (int)(b.len >> 4)) dfl_block_huff<0>(w, isEof, blk, b.len, last);
        else dfl_block_dynamic<0>(w, s, toks, isEof, blk, b.len, last);
    }
    if (ends) {
        if (eof && n == 0) { w.stored_header(0, true); w.flush(); }
        else {
            if (!eof) w.stored_header(0, false);
            w.flush();
        }
        if (P.format == DFL_FMT_GZIP) { w.stored_header(0, true); w.flush(); }   // Close: StatelessDeflate(nil, true)
        P.out_sizes[i] = w.overflow ? -4 : (int64_t)w.n;
    } else {
        st->bits = w.bits; st->n = w.n; st->nbits = w.nbits; st->overflow = w.overflow;
        st->lastHeader = w.lastHeader; st->lastHuffMan = w.lastHuffMan; st->litSel = w.litSel;
    }
}

// One warp: the CRC-32 of input i folded onto its seed (gzip: the member's CRC-32 and ISIZE after the stream)
B2C_DEV void dfl_crc_warp(const DflParams &P, uint32_t i, const uint32_t *tab, unsigned lane) {
    const uint32_t n = P.src_sizes[i];
    if (dfl_too_big(P, i)) return;
    uint32_t c = inf_crc32_warp(dfl_src(P, i), n, tab, lane);
    const uint32_t seed = P.crc_in ? P.crc_in[i] : 0;
    if (seed) c ^= inf_crc_multmodp(inf_crc_xpow8(n), seed);
    if (lane != 0) return;
    if (P.crc_out) P.crc_out[i] = c;
    if (P.format != DFL_FMT_GZIP) return;
    const int64_t r = P.out_sizes[i];
    if (r < 0) return;
    if ((uint64_t)r + 8 > dfl_cap(P, i)) { P.out_sizes[i] = -4; return; }
    uint8_t *o = dfl_dst(P, i) + r;
    for (int k = 0; k < 4; k++) { o[k] = (uint8_t)(c >> (8 * k)); o[4 + k] = (uint8_t)(n >> (8 * k)); }
    P.out_sizes[i] = r + 8;
}

// ---- BestSpeed: flate.NewWriter(w, BestSpeed) for Writes then Close (deflate.go:713-880, level1.go, fast_encoder.go),
// raw or inside the zlib / gzip writers' framing, one lane per input.
// The compressor fills a 65 535-byte window and runs storeFast each time it is full and more bytes arrive; Close runs it
// once more with sync set (deflate.go:755-770, :865-880).  Without Flush the blocks therefore depend on the byte count
// alone: consecutive 65 535-byte windows, the last one possibly shorter and the only one written with sync.  fastEncL1
// parses each window with the table and history the windows before it left, so parse and bit writer share the lane.
constexpr int32_t DFL_L1_WINDOW = 65535;               // maxStoreBlockSize; also e.cur's start
constexpr int32_t DFL_L1_HIST = 5 * DFL_L1_WINDOW;     // allocHistory: cap(e.hist)
constexpr int32_t DFL_L1_MAXOFF = 32768;               // maxMatchOffset
constexpr uint32_t DFL_L1_TABLE = 1u << 15;            // tableSize, int32 entries
constexpr uint32_t DFL_L1_TOKENS = 65536;              // tokens of one window: at most one per byte
constexpr int DFL_FMT_ZLIB = 1;
// The input cap.  The table holds e.cur + hist position; e.cur starts at 65 535 and grows only when addBlock moves the
// history down, by at most the bytes added, so it stays <= 65 535 + n.  With n <= 2^30 that is below bufferReset
// (2^31 - 6 * 65 535 - 1, fast_encoder.go:49), Encode's table shift (level1.go:29-49) never runs, and every position
// below fits an int32.
constexpr uint32_t DFL_L1_MAX_INPUT = 1u << 30;
// The 16-bit counts of DflSlot and DflState cannot overflow: a window has at most 65 535 bytes and every token covers at
// least one of them, so litHist / extraHist / offHist, and literalFreq / offsetFreq built from them, count at most 65 535
// (the EOB and the empty-offset 1 have slots of their own); writeBlockHuff's literalFreq counts the window's bytes, at most
// 65 535 per value; codegenFreq counts at most 320 code lengths.  The reference keeps the same uint16 counts.

// Little-endian 8 bytes at p from the aligned words that hold them.  The second word is read only when p is unaligned,
// and then it holds p[7]: no load touches a word outside the bytes asked for.
B2C_DEV uint64_t dfl_ld64u(const uint8_t *p) {
    const uintptr_t a = reinterpret_cast<uintptr_t>(p);
    const uint64_t *w = reinterpret_cast<const uint64_t *>(a & ~(uintptr_t)7);
    const uint32_t sh = (uint32_t)(a & 7) * 8;
    const uint64_t lo = w[0];
    return sh ? (lo >> sh) | (w[1] << (64 - sh)) : lo;
}
B2C_DEV uint32_t dfl_l1_hash(uint64_t u) { return (uint32_t)(((u << 24) * 889523592379ull) >> 49); }  // hashLen(u, 15, 5)
// matchLen(in[a:end], in[b:]) (matchlen_generic.go), b < a
B2C_DEV int32_t dfl_l1_matchlen(const uint8_t *in, int32_t a, int32_t b, int32_t end) {
    int32_t k = 0;
    for (; a + k + 8 <= end; k += 8) {
        const uint64_t x = dfl_ld64u(in + a + k) ^ dfl_ld64u(in + b + k);
        if (x) return k + (__ffsll((long long)x) - 1) / 8;
    }
    while (a + k < end && in[a + k] == in[b + k]) k++;
    return k;
}

// fastEncL1.Encode (level1.go:51-215) of the window in[bs, be) whose e.hist starts at in[hs] (addBlock,
// fast_encoder.go:81-101).  The input is read in place: positions are the input's, and a table entry e.cur + hist position
// is 65 535 + input position, since e.cur - hs starts at 65 535 and a move adds the same shift to both.  e.hist's bounds
// are kept exactly: backward extension stops at hs (`t > 0`), and matches end at be (e.hist ends with the window).
B2C_DEV void dfl_l1_parse(const uint8_t *in, int32_t hs, int32_t bs, int32_t be, DflTok &dst, int32_t *table) {
    const int32_t sLimit = be - 11;                    // len(src) - inputMargin
    int32_t s = bs, nextEmit = bs, nextS, t;
    uint64_t cv = dfl_ld64u(in + s);
    for (;;) {
        for (;;) {                                     // two probes per step, skipping faster the longer nothing matches
            uint32_t nextHash = dfl_l1_hash(cv);
            int32_t candidate = table[nextHash];
            nextS = s + 2 + ((s - nextEmit) >> 5);
            if (nextS > sLimit) goto emitRemainder;
            uint64_t now = dfl_ld64u(in + nextS);
            table[nextHash] = s + DFL_L1_WINDOW;
            nextHash = dfl_l1_hash(now);
            t = candidate - DFL_L1_WINDOW;
            if (s - t < DFL_L1_MAXOFF && (uint32_t)cv == (uint32_t)dfl_ld64u(in + t)) {
                table[nextHash] = nextS + DFL_L1_WINDOW;
                break;
            }
            cv = now;
            s = nextS;
            nextS++;
            candidate = table[nextHash];
            now >>= 8;
            table[nextHash] = s + DFL_L1_WINDOW;
            t = candidate - DFL_L1_WINDOW;
            if (s - t < DFL_L1_MAXOFF && (uint32_t)cv == (uint32_t)dfl_ld64u(in + t)) {
                table[nextHash] = nextS + DFL_L1_WINDOW;
                break;
            }
            cv = now;
            s = nextS;
        }
        for (;;) {
            int32_t l = dfl_l1_matchlen(in, s + 4, t + 4, be) + 4;
            while (t > hs && s > nextEmit && in[t - 1] == in[s - 1]) { s--; t--; l++; }
            for (int32_t k = nextEmit; k < s; k++) dst.lit(in[k]);
            dst.match_long(l, (uint32_t)(s - t - 1)); // the inlined AddMatchLong: lengths above 258 split
            s += l;
            nextEmit = s;
            if (nextS >= s) s = nextS + 1;
            if (s >= sLimit) {
                if (s + l + 8 < be) table[dfl_l1_hash(dfl_ld64u(in + s))] = s + DFL_L1_WINDOW;
                goto emitRemainder;
            }
            uint64_t x = dfl_ld64u(in + s - 2);
            const int32_t o = DFL_L1_WINDOW + s - 2;
            table[dfl_l1_hash(x)] = o;
            x >>= 16;
            const uint32_t currHash = dfl_l1_hash(x);
            const int32_t candidate = table[currHash];
            table[currHash] = o + 2;
            t = candidate - DFL_L1_WINDOW;
            if (s - t > DFL_L1_MAXOFF || (uint32_t)x != (uint32_t)dfl_ld64u(in + t)) { cv = x >> 8; s++; break; }
        }
    }
emitRemainder:
    if (nextEmit < be && dst.s->n != 0)
        for (int32_t k = nextEmit; k < be; k++) dst.lit(in[k]);
}

// An input the BestSpeed lane refuses (B2C_ERR_ARG): over src_stride, or over the cap
B2C_DEV bool dfl_l1_refused(const DflParams &P, uint32_t i) {
    return dfl_too_big(P, i) || P.src_sizes[i] > DFL_L1_MAX_INPUT;
}

// One lane: input i as one member of P.format, written as the reference's writers write it for Writes then Close.  slot:
// the lane's scratch (a zeroed table of DFL_L1_TABLE entries, DFL_L1_TOKENS tokens, a DflSlot and a DflState).  Result:
// out_sizes[i] = the member's bytes before its trailer (the check kernel appends it), B2C_ERR_DST_SMALL or B2C_ERR_ARG.
B2C_DEV void dfl_l1_lane(const DflParams &P, uint32_t i, uint32_t slot, int32_t *table) {
    if (dfl_l1_refused(P, i)) { P.out_sizes[i] = DFL_ERR_ARG; return; }
    const int32_t n = (int32_t)P.src_sizes[i];
    const uint8_t *in = dfl_src(P, i);
    DflSlot *sl = P.slots + slot;
    DflTok tok{sl, P.tokens + (size_t)slot * DFL_L1_TOKENS};
    DflWriter w;
    w.st = P.state + slot; w.out = dfl_dst(P, i); w.cap = dfl_cap(P, i);
    w.bits = 0; w.n = 0; w.nbits = 0; w.overflow = false; w.lastHeader = 0; w.lastHuffMan = 0; w.litSel = 0;
    if (P.format == DFL_FMT_ZLIB) { w.byte(0x78); w.byte(0x01); }   // zlib/writer.go:95-130 at BestSpeed
    for (uint32_t k = 0; k < P.hlen; k++) w.byte(P.hdr[k]);
    int32_t hs = 0, hl = 0;                            // e.hist: its start in the input and its length
    for (int32_t bs = 0; bs < n && !w.overflow;) {     // storeFast (deflate.go:713-751) per window
        const int32_t len = n - bs < DFL_L1_WINDOW ? n - bs : DFL_L1_WINDOW, be = bs + len;
        const bool sync = be == n;                     // the window Close stores
        const uint8_t *blk = in + bs;
        if (len < 128) {                               // only the last window is ever short
            if (len <= 32) w.stored(blk, (uint32_t)len, false);
            else dfl_block_huff<7>(w, false, blk, (uint32_t)len, true);
            break;
        }
        if (hl + len > DFL_L1_HIST && hl > 0) { hs += hl - DFL_L1_MAXOFF; hl = DFL_L1_MAXOFF; }   // addBlock's move
        hl += len;
        for (uint32_t k = 0; k < sizeof(DflSlot) / 4; k++) reinterpret_cast<uint32_t *>(sl)[k] = 0;
        dfl_l1_parse(in, hs, bs, be, tok, table);
        if (sl->n == 0) w.stored(blk, (uint32_t)len, false);
        else if ((int)sl->n > len - (len >> 4)) dfl_block_huff<7>(w, false, blk, (uint32_t)len, sync);
        else dfl_block_dynamic<7>(w, sl, tok.t, false, blk, (uint32_t)len, sync);
        bs = be;
    }
    w.stored_header(0, true);                          // close: writeStoredHeader(0, true), flush
    w.flush();
    P.out_sizes[i] = w.overflow ? -4 : (int64_t)w.n;
}

// One warp: input i's CRC-32 (raw, gzip) or Adler-32 (zlib) to crc_out, and the trailer: gzip CRC-32 and ISIZE
// (gzip/gzip.go:264-290), zlib the Adler-32 big-endian (zlib/writer.go:170-195).  Raw without crc_out has nothing to do.
B2C_DEV void dfl_l1_check_warp(const DflParams &P, uint32_t i, const uint32_t *tab, unsigned lane) {
    if (dfl_l1_refused(P, i) || (P.format == DFL_FMT_RAW && !P.crc_out)) return;
    const uint32_t n = P.src_sizes[i];
    const uint8_t *in = dfl_src(P, i);
    const uint32_t c = P.format == DFL_FMT_ZLIB ? inf_adler32_warp(in, n, lane) : inf_crc32_warp(in, n, tab, lane);
    if (lane != 0) return;
    if (P.crc_out) P.crc_out[i] = c;
    const int64_t r = P.out_sizes[i];
    if (P.format == DFL_FMT_RAW || r < 0) return;
    const uint32_t tl = P.format == DFL_FMT_GZIP ? 8 : 4;
    if ((uint64_t)r + tl > dfl_cap(P, i)) { P.out_sizes[i] = -4; return; }
    uint8_t *o = dfl_dst(P, i) + r;
    if (P.format == DFL_FMT_GZIP)
        for (int k = 0; k < 4; k++) { o[k] = (uint8_t)(c >> (8 * k)); o[4 + k] = (uint8_t)(n >> (8 * k)); }
    else
        for (int k = 0; k < 4; k++) o[k] = (uint8_t)(c >> (24 - 8 * k));
    P.out_sizes[i] = r + tl;
}

// ---- HuffmanOnly (-2, ConstantCompression) and NoCompression (0): flate.NewWriter(w, level) for Writes then Close
// (deflate.go:683-708, :755-827, :865-880), raw or inside the zlib / gzip writers' framing, every window in parallel.
// Neither level has a match finder.  The compressor fills a window (32 768 bytes at -2, 65 535 at 0) and writes it as one
// block each time it is full and more bytes arrive; Close writes the last one with sync, then writeStoredHeader(0, true).
// Without Flush the windows depend on the byte count alone, and all one window passes to the next is the bit writer's
// table reuse: lastHeader and the table in force.  So the work splits into four passes over a batch:
//   analysis: one CTA per window: its histogram (shared-memory atomics), its checksum term, writeBlockHuff's float64
//             test, its own table (generate over 257 symbols) with that table's canReuseBits and dynamic header.
//   plan:     one warp per input walks its windows in order through writeBlockHuff's reuse decisions -- the reuse cost is
//             a warp dot product -- and records each window's outcome, owed EOB and bit range; then it sums the member's
//             size and, if it fits, writes the header, the close block and the trailer.  Level 0 stores every window:
//             the ranges are closed-form and no walk runs.
//   emit:     one CTA per window writes the bytes its bit range covers whole; the partial first and last bytes it
//             shares with its neighbours go to its record.
//   finish:   one thread per window writes the byte in which its range ends, from the pieces of every range in it.
// Every output byte is written by one thread, and nothing at all for an input whose member does not fit its capacity.
constexpr uint32_t DFL_NOLZ_WINDOW_HUFF = 32768, DFL_NOLZ_WINDOW_STORE = 65535;
constexpr int DFL_NOLZ_PEN = 10;                       // logNewTablePenalty of ConstantCompression
constexpr uint32_t DFL_NOLZ_STORED = 0xffffffffu;
constexpr int DFL_NOLZ_THREADS = 256;
// A Huffman window's bits: the owed EOB (<= 15), then a new table's header (<= 17 + 19 * 3 + 258 * 7 = 1 880) and
// canReuseBits of its own table, EOB included, or the reused table's codes and EOB.  Both code parts are below the stored
// size (len + 5) * 8 <= 262 184 (estBits counts them and is below it), so with the 7-bit offset of the first bit the
// staging holds at most 7 + 15 + 1 880 + 262 183 bits: 8 253 words.
constexpr uint32_t DFL_NOLZ_STAGE_WORDS = 8256;

struct DflNolzWin {                                    // one window's record (slot = pass input * max_windows + k)
    uint32_t check[2];                                 // analysis: its checksum term (dfl_nolz_analyse)
    int32_t est, hdr;                                  // analysis: own table's canReuseBits (-1: stored by the float64
                                                       // test) and its header's bits
    uint64_t bit, end;                                 // plan: its bit range in the stream
    uint32_t eob, use;                                 // plan: the EOB code it owes first (0: none); DFL_NOLZ_STORED
                                                       // or the window whose table codes its bytes
    uint32_t sync, pieces;                             // plan: it is the last window; emit: its partial first byte |
                                                       // its partial last byte << 8
    uint16_t hist[256];
    uint32_t codes[260];                               // own table, 257 codes
    uint8_t hbits[240];                                // own table's dynamic header, LSB first, zero after its bits
};

struct DflNolzParams {
    const uint8_t *src_base; size_t src_stride; const uint64_t *src_offsets; const uint32_t *src_sizes;
    uint8_t *dst_base; size_t dst_stride; const uint64_t *dst_offsets; uint32_t dst_cap; const uint32_t *dst_caps;
    int64_t *out_sizes; uint32_t *crc_out;
    const uint8_t *hdr; uint32_t hlen;
    int format, level;
    uint32_t max_windows, i0, i1;                      // the inputs of this pass
    DflNolzWin *wins;                                  // the pass's records
};

__host__ __device__ inline uint32_t dfl_nolz_window(int level) {
    return level == 0 ? DFL_NOLZ_WINDOW_STORE : DFL_NOLZ_WINDOW_HUFF;
}
__host__ __device__ inline uint32_t dfl_nolz_windows(uint64_t n, int level) {
    return (uint32_t)((n + dfl_nolz_window(level) - 1) / dfl_nolz_window(level));
}
B2C_DEV const uint8_t *dfl_nolz_src(const DflNolzParams &P, uint32_t i) {
    return P.src_base + (P.src_offsets ? P.src_offsets[i] : (uint64_t)i * P.src_stride);
}
B2C_DEV uint8_t *dfl_nolz_dst(const DflNolzParams &P, uint32_t i) {
    return P.dst_base + (P.dst_offsets ? P.dst_offsets[i] : (uint64_t)i * P.dst_stride);
}
// the stream's first byte in the member: after 78 01 (zlib) or the gzip header
B2C_DEV uint32_t dfl_nolz_hoff(const DflNolzParams &P) {
    return P.format == DFL_FMT_ZLIB ? 2 : (P.format == DFL_FMT_GZIP ? P.hlen : 0);
}
B2C_DEV bool dfl_nolz_refused(const DflNolzParams &P, uint32_t i) { return P.src_stride && P.src_sizes[i] > P.src_stride; }
B2C_DEV bool dfl_nolz_checked(const DflNolzParams &P) { return P.format != DFL_FMT_RAW || P.crc_out; }

// Slot g of the pass: input i, window k of nw; false for a slot past the input's windows or of a refused input
struct DflNolzSlot { uint32_t i, k, n, nw; };
B2C_DEV bool dfl_nolz_slot(const DflNolzParams &P, uint64_t g, DflNolzSlot &s) {
    s.i = P.i0 + (uint32_t)(g / P.max_windows); s.k = (uint32_t)(g % P.max_windows);
    if (s.i >= P.i1 || dfl_nolz_refused(P, s.i)) return false;
    s.n = P.src_sizes[s.i]; s.nw = dfl_nolz_windows(s.n, P.level);
    return s.k < s.nw;
}

// The checksum of an input of n bytes is a sum of terms, one per piece [a, b) of it, so the pieces are independent:
//  - CRC-32: crc(A || B) = crc(A) * x^(8|B|) ^ crc(B) (mod P), so crc = XOR over the pieces of crc(piece) * x^(8 (n - b)).
//  - Adler-32 with s1 = 1 + the bytes, s2 = the sum of the running s1: s1 = 1 + sum of the pieces' byte sums a, and
//    s2 = n + sum of (the piece's own s2 from zero) + (n - b) * a.  A term is (a, that s2 part) mod 65 521.
constexpr uint32_t DFL_ADLER_MOD = 65521;
B2C_DEV void dfl_nolz_check_term(const DflNolzParams &P, const uint8_t *p, uint32_t len, uint32_t after, const uint32_t *tab,
                                 unsigned lane, uint32_t *t) {
    if (P.format == DFL_FMT_ZLIB) {
        const uint32_t v = inf_adler32_warp(p, len, lane);
        const uint32_t a = ((v & 0xffff) + DFL_ADLER_MOD - 1) % DFL_ADLER_MOD;
        const uint32_t b = ((v >> 16) + DFL_ADLER_MOD - len % DFL_ADLER_MOD) % DFL_ADLER_MOD;
        t[0] = a;
        t[1] = (uint32_t)(((uint64_t)(after % DFL_ADLER_MOD) * a + b) % DFL_ADLER_MOD);
    } else {
        const uint32_t c = inf_crc32_warp(p, len, tab, lane);
        t[0] = c ? inf_crc_multmodp(inf_crc_xpow8(after), c) : 0;
        t[1] = 0;
    }
}
B2C_DEV void dfl_nolz_check_add(const DflNolzParams &P, uint32_t *acc, const uint32_t *t) {
    if (P.format == DFL_FMT_ZLIB) {
        acc[0] = (acc[0] + t[0]) % DFL_ADLER_MOD;
        acc[1] = (acc[1] + t[1]) % DFL_ADLER_MOD;
    } else {
        acc[0] ^= t[0];
    }
}

// analysis: one CTA of DFL_NOLZ_THREADS per window slot g.  Shared: st (a writer state for generate / the header),
// hist[256], terms[2 * DFL_NOLZ_THREADS / 32], tab (the CRC-32 table).  Level 0 needs the checksum term only.
B2C_DEV void dfl_nolz_analyse(const DflNolzParams &P, uint64_t g, DflState *st, uint32_t *hist, uint32_t *terms,
                              const uint32_t *tab, unsigned tid) {
    DflNolzSlot s;
    if (!dfl_nolz_slot(P, g, s)) return;
    const uint32_t W = dfl_nolz_window(P.level), ws = s.k * W, len = s.n - ws < W ? s.n - ws : W;
    const uint8_t *in = dfl_nolz_src(P, s.i) + ws;
    DflNolzWin *r = P.wins + g;
    const bool huff = P.level != 0;
    if (huff) for (uint32_t t = tid; t < 256; t += DFL_NOLZ_THREADS) hist[t] = 0;
    __syncthreads();
    if (huff) for (uint32_t b = tid; b < len; b += DFL_NOLZ_THREADS) atomicAdd(&hist[in[b]], 1u);
    if (dfl_nolz_checked(P)) {                         // each warp one eighth of the window
        constexpr uint32_t NWARP = DFL_NOLZ_THREADS / 32;
        const uint32_t w = tid >> 5, sub = (len + NWARP - 1) / NWARP;
        const uint32_t lo = w * sub < len ? w * sub : len, hi = lo + sub < len ? lo + sub : len;
        uint32_t t[2];
        dfl_nolz_check_term(P, in + lo, hi - lo, s.n - ws - hi, tab, tid & 31, t);
        if ((tid & 31) == 0) { terms[2 * w] = t[0]; terms[2 * w + 1] = t[1]; }
        __syncthreads();
        if (tid == 0) {
            uint32_t acc[2] = {0, 0};
            for (uint32_t k = 0; k < NWARP; k++) dfl_nolz_check_add(P, acc, terms + 2 * k);
            r->check[0] = acc[0]; r->check[1] = acc[1];
        }
    }
    if (!huff) return;
    __syncthreads();
    uint16_t *lf = st->literalFreq;
    for (uint32_t t = tid; t < 256; t += DFL_NOLZ_THREADS) { lf[t] = (uint16_t)hist[t]; r->hist[t] = (uint16_t)hist[t]; }
    __syncthreads();
    if (tid == 0) {                                    // writeBlockHuff's per-window part (window <= 32 768: storable)
        if (len > 1024 && dfl_huff_incompressible(lf, len)) {
            r->est = -1; r->hdr = 0;
        } else {
            lf[DFL_EOB] = 1;
            dfl_generate(&st->lit[0], lf, DFL_EOB + 1, 15);
            r->est = dfl_reuse_bits(st->lit[0].codes, lf, DFL_EOB + 1);
            DflWriter w;
            w.st = st; w.out = r->hbits; w.cap = sizeof(r->hbits);
            w.bits = 0; w.n = 0; w.nbits = 0; w.overflow = false; w.lastHeader = 0; w.lastHuffMan = 0; w.litSel = 0;
            const uint32_t huffOff[1] = {dfl_hcode(0, 1)};
            w.gen_codegen(DFL_EOB + 1, 1, st->lit[0].codes, huffOff);
            dfl_generate(&st->cg, st->codegenFreq, DFL_CG, 7);
            r->hdr = w.header_size();
            w.dynamic_header(DFL_EOB + 1, 1, w.codegens(), false);
            if (w.nbits) w.byte((uint8_t)w.bits);
            for (uint64_t j = w.n; j < sizeof(r->hbits); j++) r->hbits[j] = 0;
        }
    }
    __syncthreads();
    if (r->est >= 0)
        for (uint32_t t = tid; t <= DFL_EOB; t += DFL_NOLZ_THREADS) r->codes[t] = st->lit[0].codes[t];
}

// plan, level -2: writeBlockHuff's decisions for the windows of an input of n bytes, in order, on one warp.  Lane l holds
// the table in force's codes for bytes 8l .. 8l + 7; the next window's fields are loaded while this one is decided.
B2C_DEV void dfl_nolz_walk(DflNolzWin *R, uint32_t nw, uint32_t n, unsigned lane) {
    int L = 0;                                         // lastHeader
    uint32_t t = 0, teob = 0, tc[8];                   // the table in force: its window, EOB code, this lane's codes
    for (int j = 0; j < 8; j++) tc[j] = 0;
    uint64_t p = 0;
    int nest = R[0].est, nhdr = R[0].hdr;
    uint4 nh = reinterpret_cast<const uint4 *>(R[0].hist)[lane];
    for (uint32_t k = 0; k < nw; k++) {
        DflNolzWin *r = R + k;
        const int est0 = nest, hdr = nhdr;
        const uint4 h = nh;
        if (k + 1 < nw) { nest = R[k + 1].est; nhdr = R[k + 1].hdr; nh = reinterpret_cast<const uint4 *>(R[k + 1].hist)[lane]; }
        const uint32_t len = k + 1 < nw ? DFL_NOLZ_WINDOW_HUFF : n - k * DFL_NOLZ_WINDOW_HUFF;
        const bool sync = k + 1 == nw;
        bool stored = est0 < 0;
        int est = 0;
        if (!stored) {
            est = est0 + (L ? L : 70 * 8);
            est += est >> DFL_NOLZ_PEN;
            stored = (int)(len + 5) * 8 <= est;
        }
        uint32_t eob = 0, use = DFL_NOLZ_STORED;
        uint64_t bits;
        if (stored) {                                  // writeStoredHeader: the owed EOB, 3 bits, the byte's end, LEN/NLEN
            if (L > 0) eob = teob;
            L = 0;
            bits = (((p + (eob & 0xff) + 3 + 7) & ~7ull) - p) + 32 + 8 * (uint64_t)len;
        } else {
            int reuse = 0x7fffffff;
            if (L > 0) {                               // canReuseBits(table in force, literalFreq[:256])
                const uint32_t hw[4] = {h.x, h.y, h.z, h.w};
                int part = 0;
                bool miss = false;
                for (int j = 0; j < 8; j++) {
                    const uint32_t f = (hw[j >> 1] >> (16 * (j & 1))) & 0xffff;
                    if (f) { miss = miss || tc[j] == 0; part += (int)f * (int)(tc[j] & 0xff); }
                }
                for (int o = 16; o; o >>= 1) part += __shfl_xor_sync(FULLMASK, part, o);
                reuse = __any_sync(FULLMASK, miss) ? 0x7fffffff : part;
                if (est < reuse) { eob = teob; L = 0; }
            }
            if (L == 0) {                              // a new table: this window's
                t = k; L = hdr;
                const uint4 a = reinterpret_cast<const uint4 *>(r->codes)[2 * lane],
                            b = reinterpret_cast<const uint4 *>(r->codes)[2 * lane + 1];
                tc[0] = a.x; tc[1] = a.y; tc[2] = a.z; tc[3] = a.w; tc[4] = b.x; tc[5] = b.y; tc[6] = b.z; tc[7] = b.w;
                teob = r->codes[DFL_EOB];
                bits = (uint64_t)hdr + est0 - (teob & 0xff);
            } else {
                bits = (uint64_t)reuse;
            }
            use = t;
            bits += eob & 0xff;
            if (sync) { bits += teob & 0xff; L = 0; }
        }
        if (lane == 0) { r->bit = p; r->end = p + bits; r->eob = eob; r->use = use; r->sync = sync; }
        p += bits;
    }
}

// plan: one warp per input of the pass.  The member's size, B2C_ERR_DST_SMALL if it does not fit (nothing is written),
// else the header, the close block's bytes after the one a window shares, the trailer and the checksum.
B2C_DEV void dfl_nolz_plan_warp(const DflNolzParams &P, uint32_t i, unsigned lane) {
    if (dfl_nolz_refused(P, i)) { if (lane == 0) P.out_sizes[i] = DFL_ERR_ARG; return; }
    const uint32_t n = P.src_sizes[i], nw = dfl_nolz_windows(n, P.level);
    DflNolzWin *R = P.wins + (uint64_t)(i - P.i0) * P.max_windows;
    uint32_t acc[2] = {0, 0};
    if (dfl_nolz_checked(P)) {
        for (uint32_t k = lane; k < nw; k += 32) dfl_nolz_check_add(P, acc, R[k].check);
        for (int o = 16; o; o >>= 1) {
            const uint32_t t[2] = {__shfl_xor_sync(FULLMASK, acc[0], o), __shfl_xor_sync(FULLMASK, acc[1], o)};
            dfl_nolz_check_add(P, acc, t);
        }
    }
    const uint32_t check = P.format == DFL_FMT_ZLIB ? ((acc[1] + n % DFL_ADLER_MOD) % DFL_ADLER_MOD) << 16 | (acc[0] + 1) % DFL_ADLER_MOD
                                                     : acc[0];
    uint64_t sc;                                       // the close block's first bit
    if (P.level == 0) {                                // every window stored: len + 5 bytes, byte-aligned
        for (uint32_t k = lane; k < nw; k += 32) {
            const uint32_t len = k + 1 < nw ? DFL_NOLZ_WINDOW_STORE : n - k * DFL_NOLZ_WINDOW_STORE;
            DflNolzWin *r = R + k;
            r->bit = (uint64_t)k * (DFL_NOLZ_WINDOW_STORE + 5) * 8; r->end = r->bit + (uint64_t)(len + 5) * 8;
            r->eob = 0; r->use = DFL_NOLZ_STORED; r->sync = k + 1 == nw;
        }
        sc = (uint64_t)n + 5ull * nw;
        sc *= 8;
    } else {
        if (nw) dfl_nolz_walk(R, nw, n, lane);
        __syncwarp();
        sc = nw ? R[nw - 1].end : 0;
    }
    const uint32_t hoff = dfl_nolz_hoff(P), tl = P.format == DFL_FMT_GZIP ? 8 : (P.format == DFL_FMT_ZLIB ? 4 : 0);
    const uint64_t cend = (sc + 10 + 7) >> 3, total = hoff + cend + tl;
    if (total > (P.dst_caps ? P.dst_caps[i] : P.dst_cap)) { if (lane == 0) P.out_sizes[i] = -4; return; }
    uint8_t *o = dfl_nolz_dst(P, i);
    if (P.format == DFL_FMT_ZLIB) { if (lane < 2) o[lane] = lane ? 0x01 : 0x78; }   // zlib/writer.go:95-130 at -2 / 0
    else for (uint32_t k = lane; k < hoff; k += 32) o[k] = P.hdr[k];
    // writeStoredHeader(0, true): the fixed header 011 then 7 zero bits, then the byte's end.  Its first byte is a
    // window's last when the block does not start a byte (the finish pass writes that one).
    const uint64_t c0 = sc >> 3;
    const uint32_t cb = 3u << (sc & 7);
    for (uint64_t b = c0 + ((sc & 7) ? 1 : 0) + lane; b < cend; b += 32) o[hoff + b] = (uint8_t)(cb >> (8 * (b - c0)));
    uint8_t *tr = o + hoff + cend;
    if (lane < 4) {
        if (P.format == DFL_FMT_GZIP) { tr[lane] = (uint8_t)(check >> (8 * lane)); tr[4 + lane] = (uint8_t)(n >> (8 * lane)); }
        else if (P.format == DFL_FMT_ZLIB) tr[lane] = (uint8_t)(check >> (24 - 8 * lane));
    }
    if (lane == 0) {
        if (P.crc_out) P.crc_out[i] = check;
        P.out_sizes[i] = (int64_t)total;
    }
}

// `nb` bits of v at bit `pos` of the staging words (v < 2^nb, nb <= 32)
B2C_DEV void dfl_nolz_or(uint32_t *stage, uint64_t pos, uint32_t v, uint32_t nb) {
    const uint32_t w = (uint32_t)(pos >> 5), sh = (uint32_t)(pos & 31);
    if (v == 0) return;
    atomicOr(&stage[w], v << sh);
    if (sh && sh + nb > 32) atomicOr(&stage[w + 1], v >> (32 - sh));
}

// emit: one CTA of DFL_NOLZ_THREADS per window slot g.  Shared: stage[DFL_NOLZ_STAGE_WORDS], codes[257],
// wsum[DFL_NOLZ_THREADS / 32].  The window's bits are ORed into the staging words at their offsets from the byte its
// range starts in, then the bytes the range covers whole go out; its partial first and last bytes go to its record.
B2C_DEV void dfl_nolz_emit(const DflNolzParams &P, uint64_t g, uint32_t *stage, uint32_t *codes, uint32_t *wsum,
                           unsigned tid) {
    DflNolzSlot s;
    if (!dfl_nolz_slot(P, g, s) || P.out_sizes[s.i] < 0) return;
    DflNolzWin *r = P.wins + g;
    const uint32_t W = dfl_nolz_window(P.level), ws = s.k * W, len = s.n - ws < W ? s.n - ws : W;
    const uint8_t *in = dfl_nolz_src(P, s.i) + ws;
    const uint64_t bit = r->bit, end = r->end, b0 = bit >> 3;
    const uint32_t rb = (uint32_t)(bit & 7), eob = r->eob, use = r->use, el = eob & 0xff;
    uint8_t *out = dfl_nolz_dst(P, s.i) + dfl_nolz_hoff(P) + b0;
    const uint8_t *sb = reinterpret_cast<const uint8_t *>(stage);
    if (use == DFL_NOLZ_STORED) {                      // the owed EOB, 3 zero bits, the byte's end, LEN / NLEN, the bytes
        const uint32_t pos = ((rb + el + 3 + 7) & ~7u) + 32;
        const uint64_t v = (uint64_t)(eob >> 8) << rb | (uint64_t)len << (pos - 32) | (uint64_t)(uint16_t)~len << (pos - 16);
        for (uint32_t j = (rb ? 1 : 0) + tid; j < pos / 8; j += DFL_NOLZ_THREADS) out[j] = (uint8_t)(v >> (8 * j));
        for (uint32_t j = tid; j < len; j += DFL_NOLZ_THREADS) out[pos / 8 + j] = in[j];
        if (tid == 0) r->pieces = rb ? (uint32_t)(v & 0xff) : 0;
        return;
    }
    const uint32_t nwords = (uint32_t)((end - 8 * b0 + 31) >> 5);
    for (uint32_t j = tid; j < nwords; j += DFL_NOLZ_THREADS) stage[j] = 0;
    const DflNolzWin *tr = P.wins + (g - s.k) + use;
    for (uint32_t j = tid; j <= DFL_EOB; j += DFL_NOLZ_THREADS) codes[j] = tr->codes[j];
    __syncthreads();
    uint64_t pos = rb;
    if (tid == 0) dfl_nolz_or(stage, pos, eob >> 8, el);
    pos += el;
    if (use == s.k) {                                  // a new table: its dynamic header
        const uint32_t hb = (uint32_t)r->hdr;
        const uint32_t *hw = reinterpret_cast<const uint32_t *>(r->hbits);
        for (uint32_t j = tid; j * 32 < hb; j += DFL_NOLZ_THREADS)
            dfl_nolz_or(stage, pos + 32 * j, hw[j], hb - 32 * j < 32 ? hb - 32 * j : 32);
        pos += hb;
    }
    // the symbols: thread t codes the bytes [t * C, (t + 1) * C), placed by a block-wide scan of their code lengths
    const uint32_t C = (len + DFL_NOLZ_THREADS - 1) / DFL_NOLZ_THREADS;
    const uint32_t lo = tid * C < len ? tid * C : len, hi = lo + C < len ? lo + C : len;
    uint32_t mine = 0;
    for (uint32_t j = lo; j < hi; j++) mine += codes[in[j]] & 0xff;
    uint32_t incl = mine;
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t v = __shfl_up_sync(FULLMASK, incl, o);
        if ((tid & 31) >= (unsigned)o) incl += v;
    }
    if ((tid & 31) == 31) wsum[tid >> 5] = incl;
    __syncthreads();
    uint64_t at = pos + incl - mine;
    for (uint32_t w = 0; w < (tid >> 5); w++) at += wsum[w];
    uint64_t acc = 0;
    uint32_t na = 0;
    for (uint32_t j = lo; j < hi; j++) {
        const uint32_t c = codes[in[j]];
        acc |= (uint64_t)(c >> 8) << na;
        na += c & 0xff;
        if (na >= 32) { dfl_nolz_or(stage, at, (uint32_t)acc, 32); at += 32; acc >>= 32; na -= 32; }
    }
    if (na) dfl_nolz_or(stage, at, (uint32_t)acc, na);
    if (tid == DFL_NOLZ_THREADS - 1 && r->sync) dfl_nolz_or(stage, at + na, codes[DFL_EOB] >> 8, codes[DFL_EOB] & 0xff);
    __syncthreads();
    const uint64_t last = (end >> 3) - b0;             // the byte the range ends in, partial when end is not aligned
    for (uint64_t j = (rb ? 1 : 0) + tid; j < last; j += DFL_NOLZ_THREADS) out[j] = sb[j];
    if (tid == 0) r->pieces = (rb ? sb[0] : 0u) | ((end & 7) ? (uint32_t)sb[last] << 8 : 0u);
}

// finish (level -2): thread for window slot g.  The byte its range ends in, when the range does not end a byte and starts
// at or before the byte's first bit: its last piece, the first pieces of the windows that start in the byte, and the
// close block's first bits when it starts there too.
B2C_DEV void dfl_nolz_finish(const DflNolzParams &P, uint64_t g) {
    DflNolzSlot s;
    if (!dfl_nolz_slot(P, g, s) || P.out_sizes[s.i] < 0) return;
    const DflNolzWin *R = P.wins + (g - s.k), *r = R + s.k;
    const uint64_t end = r->end, B = end >> 3;
    if ((end & 7) == 0 || r->bit > 8 * B) return;
    uint32_t v = r->pieces >> 8;
    uint32_t j = s.k + 1;
    for (; j < s.nw && R[j].bit < 8 * B + 8; j++) v |= R[j].pieces & 0xff;
    if (j == s.nw) {
        const uint64_t sc = R[s.nw - 1].end;
        if (sc < 8 * B + 8) v |= (3u << (sc & 7)) & 0xff;
    }
    dfl_nolz_dst(P, s.i)[dfl_nolz_hoff(P) + B] = (uint8_t)v;
}

#ifndef B2C_EMU
constexpr int DFL_PARSE_WARPS = 2, DFL_ENCODE_LANES = 64, DFL_CRC_WARPS = 4;
extern "C" __global__ void __launch_bounds__(DFL_PARSE_WARPS * 32) b2c_deflate_parse_kernel(DflParams P, uint32_t nchunks) {
    __shared__ __align__(16) int16_t table[DFL_PARSE_WARPS][1 << 13];
    const uint64_t g = P.g0 + (uint64_t)blockIdx.x * DFL_PARSE_WARPS + (threadIdx.x >> 5);
    if (g < P.g1) dfl_parse_warp(P, g, nchunks, table[threadIdx.x >> 5], threadIdx.x & 31);
}
extern "C" __global__ void __launch_bounds__(DFL_ENCODE_LANES) b2c_deflate_encode_kernel(DflParams P, uint32_t i0, uint32_t i1) {
    const uint32_t i = i0 + blockIdx.x * DFL_ENCODE_LANES + threadIdx.x;
    if (i < i1) dfl_encode_lane(P, i);
}
extern "C" __global__ void __launch_bounds__(DFL_CRC_WARPS * 32) b2c_deflate_crc_kernel(DflParams P, uint32_t nchunks) {
    __shared__ uint32_t tab[256];
    inf_crc_table(tab, threadIdx.x, blockDim.x);
    __syncthreads();
    const uint32_t i = blockIdx.x * DFL_CRC_WARPS + (threadIdx.x >> 5);
    if (i < nchunks) dfl_crc_warp(P, i, tab, threadIdx.x & 31);
}
// BestSpeed: lane i - i0 of a pass takes input i with the pass's scratch slot i - i0; tables: the pass's zeroed tables
extern "C" __global__ void __launch_bounds__(DFL_ENCODE_LANES) b2c_deflate_l1_kernel(DflParams P, int32_t *tables, uint32_t i0, uint32_t i1) {
    const uint32_t i = i0 + blockIdx.x * DFL_ENCODE_LANES + threadIdx.x;
    if (i < i1) dfl_l1_lane(P, i, i - i0, tables + (size_t)(i - i0) * DFL_L1_TABLE);
}
extern "C" __global__ void __launch_bounds__(DFL_CRC_WARPS * 32) b2c_deflate_l1_check_kernel(DflParams P, uint32_t nchunks) {
    __shared__ uint32_t tab[256];
    inf_crc_table(tab, threadIdx.x, blockDim.x);
    __syncthreads();
    const uint32_t i = blockIdx.x * DFL_CRC_WARPS + (threadIdx.x >> 5);
    if (i < nchunks) dfl_l1_check_warp(P, i, tab, threadIdx.x & 31);
}
// HuffmanOnly / NoCompression: block g of analysis and emit takes window slot g of the pass; plan: warp w takes input
// i0 + w; finish: thread g takes slot g
constexpr int DFL_NOLZ_PLAN_WARPS = 4;
extern "C" __global__ void __launch_bounds__(DFL_NOLZ_THREADS) b2c_deflate_nolz_analyse_kernel(DflNolzParams P) {
    __shared__ DflState st;
    __shared__ uint32_t hist[256], terms[2 * DFL_NOLZ_THREADS / 32], tab[256];
    inf_crc_table(tab, threadIdx.x, blockDim.x);
    dfl_nolz_analyse(P, blockIdx.x, &st, hist, terms, tab, threadIdx.x);
}
extern "C" __global__ void __launch_bounds__(DFL_NOLZ_PLAN_WARPS * 32) b2c_deflate_nolz_plan_kernel(DflNolzParams P) {
    const uint32_t i = P.i0 + blockIdx.x * DFL_NOLZ_PLAN_WARPS + (threadIdx.x >> 5);
    if (i < P.i1) dfl_nolz_plan_warp(P, i, threadIdx.x & 31);
}
extern "C" __global__ void __launch_bounds__(DFL_NOLZ_THREADS) b2c_deflate_nolz_emit_kernel(DflNolzParams P) {
    __shared__ uint32_t stage[DFL_NOLZ_STAGE_WORDS], codes[DFL_EOB + 1], wsum[DFL_NOLZ_THREADS / 32];
    dfl_nolz_emit(P, blockIdx.x, stage, codes, wsum, threadIdx.x);
}
extern "C" __global__ void __launch_bounds__(DFL_NOLZ_THREADS) b2c_deflate_nolz_finish_kernel(DflNolzParams P, uint64_t slots) {
    const uint64_t g = (uint64_t)blockIdx.x * DFL_NOLZ_THREADS + threadIdx.x;
    if (g < slots) dfl_nolz_finish(P, g);
}
#endif

}  // namespace b2c
