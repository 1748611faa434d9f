// compress_b200/csrc/b2c_inflate.cuh -- raw DEFLATE, zlib and gzip decoding (inflate) for sm_90a.
//
// What one flate.NewReader / zlib.NewReader / gzip.NewReader read to the end does (flate/inflate.go, flate/inflate_gen.go,
// zlib/reader.go, gzip/gunzip.go), for a batch of inputs.  A DEFLATE stream is serial -- every block starts at a bit
// position known only once the block before it is decoded -- so the staged shape of the S2 decoder is used, with the
// Huffman walk in front:
//   walk      one LANE per input: container headers, block headers, the dynamic tables of every block, every symbol.  The
//             lane writes each literal straight to its place in the output and one 16-byte record per match and per stored
//             run; per gzip member (zlib stream) one record of the member's output span and stored checksum.  Every
//             validity check but the checksums happens here, in stream order, so this kernel decides the outcome class.
//   exec      one WARP per input: 32 records per step; stored runs copied by the whole warp (lzc_warp_copy), then the matches
//             in dependency waves (lz_exec_match_waves).  Literals are already in place.
//   checksum  one WARP per input: CRC-32 (IEEE) or Adler-32 of every member's output, lane pieces folded, compared with the
//             stored values; then the result.  A checksum that fails comes before the walk's error, which lies after it.
//
// Decode tables.  Each lane keeps two canonical-code tables in shared memory (tree 0: the code-length code, then the
// literal/length code of the block; tree 1: the distance code): per code length L the left-justified limit of the codes
// up to L and the offset of its symbols, plus the symbols in code order -- 1088 bytes per lane with the length buffer,
// 34 KiB for the 32 lanes of a CTA, plus the fixed code's table shared by the CTA.  A symbol takes two 16-byte loads of limits, a SIMD compare of the 15-bit peek against
// all of them, and one symbol load.  The reference's reading rules are kept where they decide outcomes: a symbol is
// looked up only once maxRead bits are there (inflate.go:586-594), an empty code keeps the table of its slot (read with
// its first nine bits only, as the reference's link mask is cleared) and the distance table lives on across blocks and
// gzip members (flate's Reset keeps it), and the input running out inside the extra bits of a length or a distance ends
// a raw stream without error (inflate_gen.go:121,149,217).
#pragma once
#include "b2c_common.cuh"
#include "b2c_lz4_cvt.cuh"   // lzc_warp_copy

namespace b2c {

enum { INF_RAW = 0, INF_ZLIB = 1, INF_GZIP = 2 };
enum { INF_ERR_DST = -4, INF_ERR_CORRUPT = -5, INF_ERR_MAGIC = -7, INF_ERR_CRC = -9, INF_ERR_UNSUPPORTED = -11, INF_ERR_EOF = -12,
       INF_ERR_ARG = -102 };
enum { INF_QUIRK_EOF = 1 };                  // (internal) the reader's plain io.EOF

// Match: dst = output position, len, from = distance, kind 0.  Stored run: from = source byte offset, kind 1.
// Member (stored from the end of the input's record area): dst = first output byte, len = bytes, from = stored checksum,
// kind 0 = CRC-32, 1 = Adler-32.
struct InfRec { uint32_t dst, len, from, kind; };
struct InfHead { int32_t status; uint32_t dlen, nexec, nmem; };

struct InfParams {
    const uint8_t *src_base; uint64_t src_stride; const uint64_t *src_offsets; const uint32_t *src_sizes;
    uint8_t *dst_base; uint64_t dst_stride; const uint64_t *dst_offsets; const uint32_t *dst_caps; uint32_t dst_cap;
    int64_t *out_sizes;
    uint32_t c0, nchunks;                    // this pass: inputs c0 .. c0 + nchunks - 1
    int format, multistream;
    InfHead *heads;                          // [nchunks] of this pass
    InfRec *recs;                            // input c's area at rec_base[c] - rec_base[c0], or (c - c0) * rec_per
    const uint64_t *rec_base; uint64_t rec_per;
};

// Record bound of one input of slen bytes into cap bytes: a match takes at least 2 bits of input (a literal/length code and
// a distance code of at least one bit each) and writes at least 3 bytes; a stored run at least 5 bytes of input; a gzip
// member at least 20 (10 header, 2 deflate, 8 trailer).
__host__ __device__ inline uint64_t inf_rec_cap(uint64_t slen, uint64_t cap) {
    const uint64_t m = cap / 3 < 4 * slen ? cap / 3 : 4 * slen;
    return m + slen / 5 + slen / 18 + 2;
}

struct InfTree { uint16_t lim[16], base[16]; };
struct InfLane {
    InfTree t[2];
    uint16_t sym0[288], sym1[32];
    uint8_t len[320];
};
// The fixed literal/length code (fixedHuffmanDecoderInit, inflate.go:65-90) lives in a table of its own, one per CTA: the
// reference keeps it apart from h1, so a fixed block leaves tree 0 as it was (an empty code later reads what was there).
struct InfFixed { InfTree t; uint16_t sym[288]; };
constexpr int INF_WALK_LANES = 32;

// Builds a canonical decoding table from lens[0, n) (huffmanDecoder.init, inflate.go:116-279): false when the code is
// over- or under-subscribed (a single code of length 1 is allowed).  An empty code leaves the table as it was.
B2C_DEV bool inf_build(InfTree *t, uint16_t *sym, const uint8_t *lens, uint32_t n, uint32_t &maxRead, bool &stale) {
    uint32_t minL = 16, maxL = 0;
    for (uint32_t i = 0; i < n; i++) {
        const uint32_t l = lens[i];
        if (l) { minL = l < minL ? l : minL; maxL = l > maxL ? l : maxL; }
    }
    if (maxL == 0) { maxRead = 0; stale = true; return true; }   // empty: the reference returns before touching its chunks
    uint16_t *cnt = t->lim, *off = t->base;          // (scratch until the last loop)
    for (int L = 0; L < 16; L++) cnt[L] = 0;
    for (uint32_t i = 0; i < n; i++) cnt[lens[i]]++;
    uint32_t code = 0;
    for (uint32_t L = minL; L <= maxL; L++) code = (code << 1) + cnt[L];
    if (code != (1u << maxL) && !(code == 1 && maxL == 1)) return false;
    uint32_t o = 0;
    for (int L = 1; L < 16; L++) { off[L] = (uint16_t)o; o += cnt[L]; }
    for (uint32_t i = 0; i < n; i++) if (lens[i]) sym[off[lens[i]]++] = (uint16_t)i;
    code = 0;
    for (int L = 1; L < 16; L++) {
        code <<= 1;
        const uint32_t c = cnt[L];
        t->lim[L] = (uint16_t)((code + c) << (15 - L));
        t->base[L] = (uint16_t)(off[L] - c - code);   // symbol index = base[L] + code value
        code += c;
    }
    t->lim[0] = 0xffff;
    maxRead = minL; stale = false;
    return true;
}

// Builds the fixed code into F (len: 288 bytes of scratch).
B2C_DEV void inf_fixed_build(InfFixed *F, uint8_t *len) {
    for (uint32_t i = 0; i < 288; i++) len[i] = i < 144 ? 8 : (i < 256 ? 9 : (i < 280 ? 7 : 8));
    uint32_t maxRead;
    bool stale;
    inf_build(&F->t, F->sym, len, 288, maxRead, stale);
}

// Decodes the next symbol from bb (LSB-first, zero past the input): the symbol, *L its length (16: no code matches).
B2C_DEV uint32_t inf_decode(const InfTree *t, const uint16_t *sym, uint64_t bb, bool stale, uint32_t &L) {
    uint32_t v = __brev((uint32_t)bb) >> 17;
    if (stale) v &= 0x7fc0u;
    const uint4 a = *reinterpret_cast<const uint4 *>(t->lim), b = *reinterpret_cast<const uint4 *>(t->lim + 8);
    const uint32_t vv = v * 0x10001u;
    const uint32_t k = __popc(__vcmpgeu2(vv, a.x)) + __popc(__vcmpgeu2(vv, a.y)) + __popc(__vcmpgeu2(vv, a.z)) +
                       __popc(__vcmpgeu2(vv, a.w)) + __popc(__vcmpgeu2(vv, b.x)) + __popc(__vcmpgeu2(vv, b.y)) +
                       __popc(__vcmpgeu2(vv, b.z)) + __popc(__vcmpgeu2(vv, b.w));
    L = 1 + (k >> 4);
    if (L > 15) return 0;
    return sym[(uint16_t)(t->base[L] + (v >> (15 - L)))];
}

B2C_DEV uint32_t inf_crc_multmodp(uint32_t a, uint32_t b) {     // a * b mod P, reflected IEEE polynomial
    uint32_t m = 1u << 31, p = 0;
    for (;;) {
        if (a & m) { p ^= b; if ((a & (m - 1)) == 0) break; }
        m >>= 1;
        b = (b & 1) ? (b >> 1) ^ 0xedb88320u : b >> 1;
    }
    return p;
}
B2C_DEV uint32_t inf_crc_xpow8(uint32_t nbytes) {               // x^(8 * nbytes) mod P
    uint32_t sq = 1u << 30;
    sq = inf_crc_multmodp(sq, sq); sq = inf_crc_multmodp(sq, sq); sq = inf_crc_multmodp(sq, sq);
    uint32_t p = 1u << 31;
    for (uint32_t n = nbytes; n; n >>= 1) {
        if (n & 1) p = inf_crc_multmodp(sq, p);
        sq = inf_crc_multmodp(sq, sq);
    }
    return p;
}

struct InfWalk {
    const InfParams &P;
    const uint32_t *sw; uint32_t mis, nsw, slen;
    uint8_t *out; uint32_t cap;
    InfRec *recs; uint64_t area; uint32_t nrec, nmem;
    uint64_t bb; uint32_t nb, ip;
    uint32_t d, mstart;
    InfLane *S;
    const InfFixed *F;
    uint32_t max0, max1; bool stale0, stale1;
    bool final;

    B2C_DEV uint32_t load4(uint32_t pos) const {         // bytes pos .. pos + 3 (zero past the input)
        const uint32_t wi = (pos + mis) >> 2, sh = ((pos + mis) & 3) * 8;
        const uint32_t w0 = B2C_LDG(sw + wi), w1 = wi + 1 < nsw ? B2C_LDG(sw + wi + 1) : 0u;
        uint32_t w = __funnelshift_r(w0, w1, sh);
        const uint32_t k = slen - pos;
        if (k < 4) w &= (1u << (8 * k)) - 1;
        return w;
    }
    B2C_DEV uint32_t byte_at(uint32_t pos) const { return load4(pos) & 0xff; }
    B2C_DEV void refill() {
        if (nb <= 32 && ip < slen) {
            const uint32_t k = slen - ip < 4 ? slen - ip : 4;
            bb |= (uint64_t)load4(ip) << nb;
            nb += 8 * k; ip += k;
        }
    }
    B2C_DEV void consume(uint32_t n) { bb >>= n; nb -= n; }
    // to the next byte boundary: the bit buffer's whole bytes go back to the input
    B2C_DEV void align() { consume(nb & 7); ip -= nb >> 3; bb = 0; nb = 0; }
    B2C_DEV bool push(InfRec r) {
        if ((uint64_t)nrec + nmem >= area) return false;
        recs[nrec++] = r;
        return true;
    }
    // huffSym (inflate.go:740-790): the symbol, or a negative error
    B2C_DEV int sym_of(const InfTree *t, const uint16_t *syms, uint32_t maxRead, bool stale) {
        refill();
        if (nb < maxRead) return INF_ERR_EOF;
        uint32_t L;
        const uint32_t s = inf_decode(t, syms, bb, stale, L);
        if (L > 15) return INF_ERR_CORRUPT;
        if (L > nb) return INF_ERR_EOF;
        consume(L);
        return (int)s;
    }
    B2C_DEV int sym(int k) { return k ? sym_of(&S->t[1], S->sym1, max1, stale1) : sym_of(&S->t[0], S->sym0, max0, stale0); }
    // readHuffman, inflate.go:464-597
    B2C_DEV int read_huffman() {
        refill();
        if (nb < 14) return INF_ERR_EOF;
        const uint32_t nlit = (uint32_t)(bb & 0x1f) + 257, ndist = (uint32_t)((bb >> 5) & 0x1f) + 1, nclen = (uint32_t)((bb >> 10) & 0xf) + 4;
        if (nlit > 286 || ndist > 30) return INF_ERR_CORRUPT;
        consume(14);
        uint8_t *len = S->len;
        for (int i = 0; i < 19; i++) len[i] = 0;
        for (uint32_t i = 0; i < nclen; i++) {
            refill();
            if (nb < 3) return INF_ERR_EOF;
            len[i < 3 ? 16 + i : c_order(i - 3)] = (uint8_t)(bb & 7);
            consume(3);
        }
        if (!inf_build(&S->t[0], S->sym0, len, 19, max0, stale0)) return INF_ERR_CORRUPT;
        const uint32_t n = nlit + ndist;
        for (uint32_t i = 0; i < n;) {
            const int x = sym(0);
            if (x < 0) return x;
            if (x < 16) { len[i++] = (uint8_t)x; continue; }
            uint32_t rep, nbits, b;
            if (x == 16) {
                if (i == 0) return INF_ERR_CORRUPT;
                rep = 3; nbits = 2; b = len[i - 1];
            } else if (x == 17) { rep = 3; nbits = 3; b = 0; }
            else if (x == 18) { rep = 11; nbits = 7; b = 0; }
            else return INF_ERR_CORRUPT;      // (a stale literal table) InternalError("unexpected length code"), inflate.go:531
            refill();
            if (nb < nbits) return INF_ERR_EOF;
            rep += (uint32_t)(bb & ((1u << nbits) - 1));
            consume(nbits);
            if (i + rep > n) return INF_ERR_CORRUPT;
            for (uint32_t j = 0; j < rep; j++) len[i++] = (uint8_t)b;
        }
        const uint32_t eob = len[256];
        if (!inf_build(&S->t[0], S->sym0, len, nlit, max0, stale0) || !inf_build(&S->t[1], S->sym1, len + nlit, ndist, max1, stale1))
            return INF_ERR_CORRUPT;
        if (max0 < eob) max0 = eob;
        if (!final) max0 += 10;
        return 0;
    }
    // codeOrder[3 + j] (inflate.go:462): 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15
    B2C_DEV static uint32_t c_order(uint32_t j) { return j == 0 ? 0u : ((j & 1) ? 8 + (j >> 1) : 8 - (j >> 1)); }

    // the block decoder of inflate_gen.go:26-270 (fixed: the CTA's fixed literal/length code, 5-bit distances)
    B2C_DEV int huffman_block(bool fixed) {
        for (;;) {
            const int v = fixed ? sym_of(&F->t, F->sym, 7, false) : sym(0);
            if (v < 0) return v;
            if (v < 256) {
                if (d >= cap) return INF_ERR_DST;
                out[d++] = (uint8_t)v;
                continue;
            }
            if (v == 256) return 0;
            if (v >= 286) return INF_ERR_CORRUPT;
            // lengths 3 .. 258: codes 257 .. 264 have no extra bits, then 4 codes per extra bit, 285 = 258
            const uint32_t c = (uint32_t)v - 257;
            const uint32_t ne = (c < 8 || c == 28) ? 0u : (c - 4) >> 2;
            uint32_t length = c < 8 ? c + 3 : (c == 28 ? 258u : ((((c - 4) & 3) + 4) << ne) + 3);
            refill();                                   // (nb >= 32 or the input is used up: enough for 5 + 15 + 13 bits)
            if (ne) {
                if (nb < ne) return INF_QUIRK_EOF;
                length += (uint32_t)(bb & ((1u << ne) - 1));
                consume(ne);
            }
            uint32_t dist;
            if (fixed) {
                if (nb < 5) return INF_QUIRK_EOF;
                dist = __brev((uint32_t)bb & 0x1f) >> 27;
                consume(5);
            } else {
                const int x = sym(1);
                if (x < 0) return x;
                dist = (uint32_t)x;
            }
            if (dist >= 30) return INF_ERR_CORRUPT;
            if (dist < 4) dist++;
            else {
                const uint32_t nbits = (dist - 2) >> 1;
                const uint32_t extra = (dist & 1) << nbits;
                refill();
                if (nb < nbits) return INF_QUIRK_EOF;
                dist = (1u << (nbits + 1)) + 1 + (extra | (uint32_t)(bb & ((1u << nbits) - 1)));
                consume(nbits);
            }
            if (dist > d - mstart) return INF_ERR_CORRUPT;      // dist > dict.histSize() (dist <= 32768, the window)
            if (length > cap - d) return INF_ERR_DST;
            if (!push(InfRec{d, length, dist, 0u})) return INF_ERR_CORRUPT;   // (cannot happen: the record bound)
            d += length;
        }
    }
    // one DEFLATE stream from ip: 0 at its end, INF_QUIRK_EOF, or a negative error
    B2C_DEV int stream() {
        bb = 0; nb = 0; final = false;
        mstart = d;
        for (;;) {
            refill();
            if (nb < 3) return INF_ERR_EOF;
            final = bb & 1;
            const uint32_t typ = (uint32_t)(bb >> 1) & 3;
            consume(3);
            int r;
            if (typ == 0) {                              // dataBlock, inflate.go:600-646
                align();
                if (slen - ip < 4) return INF_ERR_EOF;
                const uint32_t w = load4(ip);
                ip += 4;
                const uint32_t n = w & 0xffff;
                if ((w >> 16) != (n ^ 0xffff)) return INF_ERR_CORRUPT;
                if (n > slen - ip || n > cap - d) return (slen - ip <= cap - d) ? (int)INF_ERR_EOF : (int)INF_ERR_DST;
                if (n && !push(InfRec{d, n, ip, 1u})) return INF_ERR_CORRUPT;
                d += n; ip += n;
                r = 0;
            } else if (typ == 1) {
                r = huffman_block(true);
            } else if (typ == 2) {
                if ((r = read_huffman())) return r;
                r = huffman_block(false);
            } else return INF_ERR_CORRUPT;
            if (r) return r;
            if (final) return 0;
        }
    }
    // gzip readHeader (gunzip.go:183-253) at ip: 0, INF_QUIRK_EOF (the reader's io.EOF) or a negative error
    B2C_DEV int gzip_header() {
        const uint32_t start = ip;
        if (slen - ip < 10) { const bool none = ip == slen; ip = slen; return none ? INF_QUIRK_EOF : INF_ERR_EOF; }
        const uint32_t w = load4(ip);
        if ((w & 0xffffff) != 0x088b1fu) return INF_ERR_MAGIC;
        const uint32_t flg = w >> 24;
        ip += 10;
        if (flg & 4) {                                   // FEXTRA
            if (slen - ip < 2) return INF_ERR_EOF;
            const uint32_t xlen = load4(ip) & 0xffff;
            ip += 2;
            if (slen - ip < xlen) return INF_ERR_EOF;
            ip += xlen;
        }
        for (uint32_t k = 8; k <= 16; k <<= 1) {          // FNAME, FCOMMENT (readString, gunzip.go:150-179)
            if (!(flg & k)) continue;
            for (uint32_t i = 0;; i++) {
                if (i >= 512) return INF_ERR_MAGIC;
                if (ip >= slen) return INF_QUIRK_EOF;
                if (byte_at(ip++) == 0) break;
            }
        }
        if (flg & 2) {                                   // FHCRC: the low half of the CRC-32 of the header so far
            if (slen - ip < 2) return INF_ERR_EOF;
            uint32_t crc = 0xffffffffu;
            for (uint32_t i = start; i < ip; i++) {
                crc ^= byte_at(i);
                for (int b = 0; b < 8; b++) crc = (crc & 1) ? (crc >> 1) ^ 0xedb88320u : crc >> 1;
            }
            if ((load4(ip) & 0xffff) != (~crc & 0xffff)) return INF_ERR_MAGIC;
            ip += 2;
        }
        if (flg >> 5) return INF_ERR_MAGIC;
        return 0;
    }
    B2C_DEV bool member(uint32_t start, uint32_t n, uint32_t sum, uint32_t adler) {
        if ((uint64_t)nrec + nmem >= area) return false;
        recs[area - 1 - nmem++] = InfRec{start, n, sum, adler};
        return true;
    }
    B2C_DEV uint32_t be32(uint32_t w) const { return __byte_perm(w, 0, 0x0123); }
    // the whole input: 0 or a negative error; nexec = the records of the members read completely
    B2C_DEV int run(uint32_t &nexec) {
        nexec = 0;
        if (P.format == INF_RAW) {
            const int r = stream();
            nexec = nrec;
            return r < 0 ? r : 0;                      // (INF_QUIRK_EOF: the content so far)
        }
        if (P.format == INF_ZLIB) {                      // zlib.Reader.Reset / Read, zlib/reader.go:93-187
            if (slen < 2) return INF_ERR_EOF;
            const uint32_t h = load4(0);
            const uint32_t cmf = h & 0xff, flg = (h >> 8) & 0xff;
            if ((cmf & 15) != 8 || (cmf >> 4) > 7 || ((cmf << 8 | flg) % 31) != 0) return INF_ERR_MAGIC;
            ip = 2;
            if (flg & 0x20) {
                if (slen < 6) return INF_ERR_EOF;
                if (be32(load4(2)) != 1) return INF_ERR_UNSUPPORTED;   // adler32 of the empty dictionary: read without one
                ip = 6;
            }
            const int r = stream();
            if (r < 0) return r;
            align();
            if (slen - ip < 4) return INF_ERR_EOF;       // (INF_QUIRK_EOF: the input is used up)
            if (!member(0, d, be32(load4(ip)), 1u)) return INF_ERR_CORRUPT;
            nexec = nrec;
            return 0;
        }
        int r = gzip_header();                           // gzip.Reader.Read, gunzip.go:256-295
        if (r) return r == INF_QUIRK_EOF ? INF_ERR_EOF : r;
        for (;;) {
            r = stream();
            if (r < 0) return r;
            align();
            if (slen - ip < 8) return INF_ERR_EOF;       // (INF_QUIRK_EOF: the input is used up)
            const uint32_t crc = load4(ip), isz = load4(ip + 4);
            ip += 8;
            if (isz != d - mstart) return INF_ERR_CRC;
            if (!member(mstart, d - mstart, crc, 0u)) return INF_ERR_CORRUPT;
            nexec = nrec;
            if (!P.multistream) return 0;
            r = gzip_header();
            if (r == INF_QUIRK_EOF) return 0;            // io.EOF: the end of the members
            if (r) return r;
        }
    }
};

B2C_DEV const uint8_t *inf_src(const InfParams &P, uint32_t c) { return P.src_base + (P.src_offsets ? P.src_offsets[c] : (uint64_t)c * P.src_stride); }
B2C_DEV uint8_t *inf_dst(const InfParams &P, uint32_t c) { return P.dst_base + (P.dst_offsets ? P.dst_offsets[c] : (uint64_t)c * P.dst_stride); }
B2C_DEV InfRec *inf_recs(const InfParams &P, uint32_t c) {
    return P.recs + (P.rec_base ? P.rec_base[c] - P.rec_base[P.c0] : (uint64_t)(c - P.c0) * P.rec_per);
}
B2C_DEV uint64_t inf_area(const InfParams &P, uint32_t c) { return P.rec_base ? P.rec_base[c + 1] - P.rec_base[c] : P.rec_per; }

// ---- walk: one lane per input
B2C_DEV void inf_walk_lane(const InfParams &P, uint32_t c, InfLane *S, const InfFixed *F) {
    const uint8_t *src = inf_src(P, c);
    const uint32_t slen = P.src_sizes[c];
    const uint32_t mis = (uint32_t)(reinterpret_cast<uintptr_t>(src) & 3);
    InfWalk W{P, reinterpret_cast<const uint32_t *>(src - mis), mis, (uint32_t)(((uint64_t)slen + mis + 3) >> 2), slen,
              inf_dst(P, c), P.dst_caps ? P.dst_caps[c] : P.dst_cap, inf_recs(P, c), inf_area(P, c), 0u, 0u,
              0ull, 0u, 0u, 0u, 0u, S, F, 0u, 0u, false, false, false};
    for (int k = 0; k < 2; k++) {                        // a code never built: no symbol matches
        S->t[k].lim[0] = 0xffff;
        for (int L = 1; L < 16; L++) S->t[k].lim[L] = 0;
    }
    uint32_t nexec = 0;
    int status = 0;
    if (!P.rec_base && slen > P.src_stride) status = INF_ERR_ARG;   // its records would not fit the room of an input
    else status = W.run(nexec);
    P.heads[c - P.c0] = InfHead{status, W.d, nexec, W.nmem};
}

// ---- exec: one warp per input, records [0, nexec)
B2C_DEV void inf_exec_warp(const InfParams &P, uint32_t c, unsigned lane) {
    const InfHead hd = P.heads[c - P.c0];
    const uint8_t *src = inf_src(P, c);
    uint8_t *out = inf_dst(P, c);
    const InfRec *recs = inf_recs(P, c);
    const uint32_t n = hd.nexec;
    InfRec next = lane < n ? recs[lane] : InfRec{0, 0, 0, 0};
    for (uint32_t base = 0; base < n; base += 32) {
        const bool mine = base + lane < n;
        const InfRec r = next;
        if (base + 32 < n) next = base + 32 + lane < n ? recs[base + 32 + lane] : InfRec{0, 0, 0, 0};
        // stored runs first (they read only the input), each by the whole warp: aligned source words, 16-byte stores
        for (unsigned m = __ballot_sync(FULLMASK, mine && r.kind == 1); m; m &= m - 1) {
            const int l = __ffs((int)m) - 1;
            const uint32_t to = __shfl_sync(FULLMASK, r.dst, l), len = __shfl_sync(FULLMASK, r.len, l), from = __shfl_sync(FULLMASK, r.from, l);
            lzc_warp_copy(out + to, src + from, len, lane);
        }
        __syncwarp();
        lz_exec_match_waves(out, mine && r.kind == 0, r.dst, r.from, r.len, lane);
    }
}

// ---- checksum: one warp per input, then the result
// CRC-32 (IEEE, reflected 0xEDB88320) of p[0, n) by one warp; result on every lane.  tab: the byte table.
B2C_DEV uint32_t inf_crc32_warp(const uint8_t *p, uint32_t n, const uint32_t *tab, unsigned lane) {
    const uint32_t seg = (((n + 31) / 32) + 3) & ~3u;
    const uint32_t lo = lane * seg < n ? lane * seg : n, hi = lo + seg < n ? lo + seg : n;
    uint32_t c = 0xffffffffu, i = lo;
    for (; i < hi && ((reinterpret_cast<uintptr_t>(p) + i) & 3); i++) c = tab[(c ^ p[i]) & 0xff] ^ (c >> 8);
    for (; i + 4 <= hi; i += 4) {
        const uint32_t w = *reinterpret_cast<const uint32_t *>(p + i);
        c = tab[(c ^ w) & 0xff] ^ (c >> 8);
        c = tab[(c ^ (w >> 8)) & 0xff] ^ (c >> 8);
        c = tab[(c ^ (w >> 16)) & 0xff] ^ (c >> 8);
        c = tab[(c ^ (w >> 24)) & 0xff] ^ (c >> 8);
    }
    for (; i < hi; i++) c = tab[(c ^ p[i]) & 0xff] ^ (c >> 8);
    c ^= 0xffffffffu;
    if (hi == lo) c = 0;
    const uint32_t pfull = inf_crc_xpow8(seg);
    uint32_t acc = 0;
    for (int l = 0; l < 32; l++) {                       // acc = acc * x^(8 |piece l|) ^ crc(piece l)
        const uint32_t cl = __shfl_sync(FULLMASK, c, l), ll = __shfl_sync(FULLMASK, hi - lo, l);
        if (l == 0) acc = cl;
        else if (ll == seg) acc = inf_crc_multmodp(pfull, acc) ^ cl;
        else if (ll) acc = inf_crc_multmodp(inf_crc_xpow8(ll), acc) ^ cl;
    }
    return acc;
}
// Adler-32 of p[0, n) by one warp: per lane s1 = sum of its bytes, s2 = sum of the running s1; pieces folded in order
// (s2 = s2a + |b| * s1a + s2b).  Result on every lane.
B2C_DEV uint32_t inf_adler32_warp(const uint8_t *p, uint32_t n, unsigned lane) {
    constexpr uint32_t M = 65521, NMAX = 5552;
    const uint32_t seg = (n + 31) / 32;
    const uint32_t lo = lane * seg < n ? lane * seg : n, hi = lo + seg < n ? lo + seg : n;
    uint32_t s1 = 0, s2 = 0;
    for (uint32_t i = lo; i < hi;) {
        const uint32_t e = hi - i > NMAX ? i + NMAX : hi;
        for (; i < e; i++) { s1 += p[i]; s2 += s1; }
        s1 %= M; s2 %= M;
    }
    uint32_t a = 0, b = 0;
    for (int l = 0; l < 32; l++) {
        const uint32_t t1 = __shfl_sync(FULLMASK, s1, l), t2 = __shfl_sync(FULLMASK, s2, l), ll = __shfl_sync(FULLMASK, hi - lo, l);
        b = (uint32_t)(((uint64_t)b + (uint64_t)(ll % M) * a + t2) % M);
        a = (a + t1) % M;
    }
    return ((b + n % M) % M) << 16 | ((a + 1) % M);
}
// the CRC-32 byte table, filled by the calling threads
B2C_DEV void inf_crc_table(uint32_t *tab, unsigned tid, unsigned nthreads) {
    for (uint32_t i = tid; i < 256; i += nthreads) {
        uint32_t v = i;
#pragma unroll
        for (int k = 0; k < 8; k++) v = (v & 1) ? (v >> 1) ^ 0xedb88320u : v >> 1;
        tab[i] = v;
    }
}
B2C_DEV void inf_check_warp(const InfParams &P, uint32_t c, const uint32_t *tab, unsigned lane) {
    const InfHead hd = P.heads[c - P.c0];
    const uint8_t *out = inf_dst(P, c);
    const InfRec *mem = inf_recs(P, c) + inf_area(P, c) - 1;
    bool bad = false;
    for (uint32_t m = 0; m < hd.nmem && !bad; m++) {
        const InfRec r = *(mem - m);
        const uint32_t v = r.kind ? inf_adler32_warp(out + r.dst, r.len, lane) : inf_crc32_warp(out + r.dst, r.len, tab, lane);
        bad = v != r.from;
    }
    if (lane == 0) P.out_sizes[c] = bad ? (int64_t)INF_ERR_CRC : (hd.status ? (int64_t)hd.status : (int64_t)hd.dlen);
}

#ifndef B2C_EMU
constexpr int INF_WARPS = 4;
extern "C" __global__ void __launch_bounds__(INF_WALK_LANES) b2c_inflate_walk_kernel(InfParams P) {
    __shared__ __align__(16) InfLane lanes[INF_WALK_LANES];
    __shared__ __align__(16) InfFixed fixed;
    if (threadIdx.x == 0) inf_fixed_build(&fixed, lanes[0].len);
    __syncthreads();
    const uint32_t i = blockIdx.x * INF_WALK_LANES + threadIdx.x;
    if (i < P.nchunks) inf_walk_lane(P, P.c0 + i, &lanes[threadIdx.x], &fixed);
}
extern "C" __global__ void __launch_bounds__(INF_WARPS * 32) b2c_inflate_exec_kernel(InfParams P) {
    const uint32_t i = blockIdx.x * INF_WARPS + (threadIdx.x >> 5);
    if (i < P.nchunks) inf_exec_warp(P, P.c0 + i, threadIdx.x & 31);
}
extern "C" __global__ void __launch_bounds__(INF_WARPS * 32) b2c_inflate_check_kernel(InfParams P) {
    __shared__ uint32_t tab[256];
    inf_crc_table(tab, threadIdx.x, blockDim.x);
    __syncthreads();
    const uint32_t i = blockIdx.x * INF_WARPS + (threadIdx.x >> 5);
    if (i < P.nchunks) inf_check_warp(P, P.c0 + i, tab, threadIdx.x & 31);
}
#endif

}  // namespace b2c
