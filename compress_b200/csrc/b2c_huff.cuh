// compress_b200/csrc/b2c_huff.cuh -- huff0 (zstd literal Huffman) on the device.
//
// Device-native replacement for the reference's
//   huff0/compress.go:43-163 (compress), :233-302 (compress1xDo / compress4X),
//   :351-385 (countSimple), :428-447 (optimalTableLog), :457-567 (buildCTable),
//   :570-607 (huffSort), :609-718 (setMaxHeight); huff0/huff0.go:180-247 (cTable.write)
//   fse/compress.go:18-78 (weights are FSE-compressed)
// One CTA cooperates on one block of literals:
//   histogram   : per-warp private bins, lanes merged with match.any (no shared atomics)
//   table build : rank-sort by all threads (same order as huffSort: count desc, symbol asc),
//                 two-queue tree by one lane (<= 255 steps, bit-exact tie-breaks), depths and the table
//                 description by one warp
//   encode      : code-length suffix sums (block scan) then every thread packs its own
//                 contiguous bit range of the 4 backward streams straight into the staging buffer.
// Output bytes are identical to the oracle's for the same literals.
#pragma once
#include "b2c_common.cuh"
#include "b2c_fse.cuh"

namespace b2c {

constexpr int HUF_TABLELOG_MAX = 11;
enum { HUF_OK = 0, HUF_INCOMPRESSIBLE = 1, HUF_USE_RLE = 2, HUF_TOO_BIG = 3 };

struct HufWork {
    uint32_t count[256];
    // sorted nodes, index +1 shifted like s.nodes (slot 0 = the "-1" sentinel)
    uint32_t ncount[514];
    uint16_t nparent[514];
    uint8_t nsym[514];
    uint8_t nbits[514];
    uint16_t ctVal[256];
    uint8_t ctBits[256];
    uint8_t weight[258];
    uint8_t tableDesc[320];
    uint32_t tableDescLen;
    uint32_t symbolLen;
    uint32_t maxCount;
    uint32_t tableLog;
    uint32_t nonNullRank;
    int32_t status;
    FseCTable wct;  // FSE table for the weights
    uint32_t scan[40];
    uint32_t streamBits[4];
    uint32_t streamBytes[4];
};

// ---------------------------------------------------------------- histogram
// whist: [nwarps][256] uint32 in shared memory.  All `nthreads` threads call.
B2C_DEV void huf_histogram(const uint8_t *in, uint32_t n, uint32_t *whist, HufWork *hw, unsigned tid,
                           unsigned nthreads, int bar_id) {
    unsigned lane = tid & 31, w = tid >> 5, nw = nthreads >> 5;
    uint32_t *h = whist + w * 256;
    for (unsigned i = lane; i < 256; i += 32) h[i] = 0;
    __syncwarp();
    for (uint32_t base = w * 32; base < n; base += nthreads) {
        uint32_t i = base + lane;
        bool valid = i < n;
        unsigned act = __ballot_sync(FULLMASK, valid);
        if (valid) {
            unsigned b = in[i];
            unsigned peers = __match_any_sync(act, b);
            if (lane == (unsigned)(__ffs((int)peers) - 1)) h[b] += (uint32_t)__popc(peers);
        }
        __syncwarp();
    }
    group_sync(bar_id, (int)nthreads);
    for (unsigned s = tid; s < 256; s += nthreads) {
        uint32_t c = 0;
        for (unsigned k = 0; k < nw; k++) c += whist[k * 256 + s];
        hw->count[s] = c;
    }
    group_sync(bar_id, (int)nthreads);
}

// ---------------------------------------------------------------- serial helpers (one thread)
B2C_DEV uint32_t huf_optimal_tablelog(uint32_t tableLogReq, uint32_t srcLen, uint32_t symbolLen) {
    uint8_t tableLog = (uint8_t)tableLogReq;
    uint32_t minBitsSrc = fse_hb(srcLen) + 1;
    uint32_t minBitsSymbols = fse_hb(symbolLen - 1) + 2;
    uint8_t minBits = (uint8_t)(minBitsSrc < minBitsSymbols ? minBitsSrc : minBitsSymbols);
    uint8_t maxBitsSrc = (uint8_t)((uint8_t)fse_hb(srcLen - 1) - 1);
    if (maxBitsSrc < tableLog) tableLog = maxBitsSrc;
    if (minBits > tableLog) tableLog = minBits;
    if (tableLog < 5) tableLog = 5;
    if (tableLog > HUF_TABLELOG_MAX) tableLog = HUF_TABLELOG_MAX;
    return tableLog;
}

B2C_DEV uint32_t huf_set_max_height(HufWork *hw, int lastNonNull, uint32_t maxNbBits) {
    uint8_t *nb = hw->nbits + 1;       // huffNode[i].nbBits
    const uint32_t *cnt = hw->ncount + 1;
    uint32_t largestBits = nb[lastNonNull];
    if (largestBits <= maxNbBits) return largestBits;
    int totalCost = 0;
    int baseCost = 1 << (largestBits - maxNbBits);
    uint32_t n = (uint32_t)lastNonNull;
    while (nb[n] > maxNbBits) {
        totalCost += baseCost - (1 << (largestBits - nb[n]));
        nb[n] = (uint8_t)maxNbBits;
        n--;
    }
    while (nb[n] == maxNbBits) n--;
    totalCost >>= (largestBits - maxNbBits);
    const uint32_t noSymbol = 0xF0F0F0F0u;
    uint32_t rankLast[HUF_TABLELOG_MAX + 2];
    for (int i = 0; i < HUF_TABLELOG_MAX + 2; i++) rankLast[i] = noSymbol;
    {
        uint32_t currentNbBits = maxNbBits;
        for (int pos = (int)n; pos >= 0; pos--) {
            if (nb[pos] >= currentNbBits) continue;
            currentNbBits = nb[pos];
            rankLast[maxNbBits - currentNbBits] = (uint32_t)pos;
        }
    }
    while (totalCost > 0) {
        uint32_t nBitsToDecrease = highbit32((uint32_t)totalCost) + 1;
        for (; nBitsToDecrease > 1; nBitsToDecrease--) {
            uint32_t highPos = rankLast[nBitsToDecrease];
            uint32_t lowPos = rankLast[nBitsToDecrease - 1];
            if (highPos == noSymbol) continue;
            if (lowPos == noSymbol) break;
            uint32_t highTotal = cnt[highPos];
            uint32_t lowTotal = 2 * cnt[lowPos];
            if (highTotal <= lowTotal) break;
        }
        while (nBitsToDecrease <= HUF_TABLELOG_MAX && rankLast[nBitsToDecrease] == noSymbol) nBitsToDecrease++;
        totalCost -= 1 << (nBitsToDecrease - 1);
        if (rankLast[nBitsToDecrease - 1] == noSymbol) rankLast[nBitsToDecrease - 1] = rankLast[nBitsToDecrease];
        nb[rankLast[nBitsToDecrease]]++;
        if (rankLast[nBitsToDecrease] == 0) {
            rankLast[nBitsToDecrease] = noSymbol;
        } else {
            rankLast[nBitsToDecrease]--;
            if (nb[rankLast[nBitsToDecrease]] != maxNbBits - nBitsToDecrease) rankLast[nBitsToDecrease] = noSymbol;
        }
    }
    while (totalCost < 0) {
        if (rankLast[1] == noSymbol) {
            while (nb[n] == maxNbBits) n--;
            nb[n + 1]--;
            rankLast[1] = n + 1;
            totalCost++;
            continue;
        }
        nb[rankLast[1] + 1]--;
        rankLast[1]++;
        totalCost++;
    }
    return maxNbBits;
}

// The 2-state encode of huf_fse_compress_weights (one thread): the weights' bitstream after the hdr NCount bytes.
B2C_DEV int huf_fse_encode_weights(const FseCTable *ct, const uint8_t *in, uint32_t n, uint32_t tableLog, uint8_t *out,
                                   uint32_t hdr) {
    // 2-state backward encode (fse/compress.go:121-205); plain LSB-first concatenation
    uint64_t acc = 0; uint32_t nacc = 0; uint32_t o = hdr;
#define WADD(val, nb)                                                                                  \
    do {                                                                                               \
        uint32_t nb__ = (nb);                                                                          \
        if (nb__) { acc |= (uint64_t)((val) & ((1u << nb__) - 1)) << nacc; nacc += nb__; }             \
        while (nacc >= 8) { out[o++] = (uint8_t)acc; acc >>= 8; nacc -= 8; }                           \
    } while (0)
#define WENC(st, sym)                                                                                  \
    do {                                                                                               \
        uint32_t s__ = (sym);                                                                          \
        uint32_t nb_ = ((st) + ct->deltaNbBits[s__]) >> 16;                                            \
        int32_t ds_ = (int32_t)((st) >> (nb_ & 15)) + (int32_t)ct->deltaFindState[s__];               \
        WADD((st), nb_);                                                                               \
        (st) = ct->stateTable[ds_];                                                                    \
    } while (0)
    uint32_t c1, c2, ip = n;
    if (ip & 1) {
        c1 = fse_init_state(ct, in[ip - 1]);
        c2 = fse_init_state(ct, in[ip - 2]);
        WENC(c1, in[ip - 3]);
        ip -= 3;
    } else {
        c2 = fse_init_state(ct, in[ip - 1]);
        c1 = fse_init_state(ct, in[ip - 2]);
        ip -= 2;
    }
    if (ip & 2) {
        WENC(c2, in[ip - 1]);
        WENC(c1, in[ip - 2]);
        ip -= 2;
    }
    while (ip >= 4) {
        WENC(c2, in[ip - 1]);
        WENC(c1, in[ip - 2]);
        WENC(c2, in[ip - 3]);
        WENC(c1, in[ip - 4]);
        ip -= 4;
    }
    WADD(c2, tableLog);
    WADD(c1, tableLog);
    WADD(1u, 1);
    if (nacc) { out[o++] = (uint8_t)acc; }
#undef WENC
#undef WADD
    if (o >= n) return -1;  // "Check if we compressed"
    return (int)o;
}

// FSE-compress the weights (fse.Compress with TableLog 6 and a supplied histogram) by one warp: normalisation and
// table fill by all lanes, the NCount and the 2-state encode on lane 0.  Every lane calls and gets the same result:
// bytes written to out or -1 (=> caller falls back to 4-bit weights).  Uses hw->nparent as table-fill scratch.
B2C_DEV int huf_fse_compress_weights(HufWork *hw, const uint8_t *in, uint32_t n, const uint32_t *hist,
                                     uint32_t symbolLen, uint32_t maxCount, uint8_t *out /* >= 300 bytes */,
                                     unsigned lane) {
    if (n <= 1) return -1;
    if (maxCount == n) return -1;                      // ErrUseRLE
    if (maxCount == 1 || maxCount < (n >> 7)) return -1;  // ErrIncompressible
    // optimalTableLog (fse/compress.go:483-508) with TableLog = 6
    uint8_t tableLog = 6;
    {
        uint32_t minBitsSrc = fse_hb(n - 1) + 1;
        uint32_t minBitsSymbols = fse_hb(symbolLen - 1) + 2;
        uint8_t minBits = (uint8_t)(minBitsSrc < minBitsSymbols ? minBitsSrc : minBitsSymbols);
        uint8_t maxBitsSrc = (uint8_t)((uint8_t)fse_hb(n - 1) - 2);
        if (maxBitsSrc < tableLog) tableLog = maxBitsSrc;
        if (minBits > tableLog) tableLog = minBits;
        if (tableLog < 5) tableLog = 5;
        if (tableLog > 12) tableLog = 12;
    }
    FseCTable *ct = &hw->wct;
    if (lane == 0) { ct->symbolLen = symbolLen; ct->tableLog = tableLog; ct->useRLE = 0; }
    ct->norm[lane] = 0; ct->norm[lane + 32] = 0;
    __syncwarp();
    if (fse_normalize(hist, symbolLen, n, tableLog, ct->norm, lane)) return -1;
    int hdr = 0;
    if (lane == 0) hdr = fse_write_ncount(ct->norm, symbolLen, tableLog, out);
    hdr = __shfl_sync(FULLMASK, hdr, 0);
    if (hdr < 0) return -1;
    if (fse_build_ctable_warp(ct, hw->nparent, lane)) return -1;
    if (n <= 2) return -1;
    int o = 0;
    if (lane == 0) o = huf_fse_encode_weights(ct, in, n, tableLog, out, (uint32_t)hdr);
    o = __shfl_sync(FULLMASK, o, 0);
    __syncwarp();
    return o;
}
// ---------------------------------------------------------------- table build (staged)
// Stage A (all threads of the group): symbolLen / maxCount / early outs, then the rank sort.
//   caller barriers: after huf_bt_stats, after huf_bt_sort.
// Stage B (one warp): tree merge (lane 0), depths, setMaxHeight, valPerRank.
// Stage C (all threads): ctBits then ctVal (barrier between the two halves is inside).
// Stage D (one warp): serialise the table (FSE-compressed or 4-bit weights).
B2C_DEV void huf_bt_stats(HufWork *hw, uint32_t n, unsigned tid) {
    if (tid < 32) {
        uint32_t m = 0, sl = 0;
        for (unsigned s = tid; s < 256; s += 32) {
            uint32_t c = hw->count[s];
            if (c) { if (c > m) m = c; sl = s + 1; }
        }
        m = warp_max(m); sl = warp_max(sl);
        if (tid == 0) {
            hw->maxCount = m; hw->symbolLen = sl;
            int st = HUF_OK;
            if (m >= n) st = (n == 1) ? HUF_INCOMPRESSIBLE : HUF_USE_RLE;
            else if (m == 1 || m < (n >> 7)) st = HUF_INCOMPRESSIBLE;
            hw->status = st;
            hw->tableDescLen = 0;
        }
    }
}
// huffSort: rank = #symbols ordered before me (count desc, symbol asc); zero counts included
B2C_DEV void huf_bt_sort(HufWork *hw, unsigned tid, unsigned nthreads) {
    uint32_t symbolLen = hw->symbolLen;
    if (nthreads == 32) {
        // one warp: bitonic sort of the 256 keys count << 8 | (255 - symbol), descending, in place in ncount[1..256]
        // (symbols >= symbolLen have count 0 and the smallest keys, so the first symbolLen slots are the ranking)
        // Only the first N = 2^ceil(log2(symbolLen)) symbols take part (>= 64): the rest have count 0 and keys below
        // every participant's, so the first symbolLen slots come out the same as from the full 256-key sort.
        uint32_t *K = hw->ncount + 1;
        unsigned N = 64;
        while (N < symbolLen) N <<= 1;
        for (unsigned s = tid; s < N; s += 32) K[s] = (hw->count[s] << 8) | (255u - s);
        __syncwarp();
        const unsigned rounds = N >> 6;                                    // pairs per lane
        for (unsigned k = 2; k <= N; k <<= 1) {
            for (unsigned j = k >> 1; j > 0; j >>= 1) {
                for (unsigned m = 0; m < rounds; m++) {
                    const unsigned t = tid + 32 * m;                       // pair index 0..N/2-1
                    const unsigned i = ((t & ~(j - 1)) << 1) | (t & (j - 1));
                    const unsigned q = i | j;
                    const uint32_t a = K[i], b = K[q];
                    const bool desc = (i & k) == 0;
                    if (desc ? (a < b) : (a > b)) { K[i] = b; K[q] = a; }
                }
                __syncwarp();
            }
        }
        for (unsigned r = tid; r < symbolLen; r += 32) {
            const uint32_t key = K[r];
            hw->nsym[1 + r] = (uint8_t)(255u - (key & 255u));
            hw->nparent[1 + r] = 0; hw->nbits[1 + r] = 0;
            K[r] = key >> 8;
        }
        for (unsigned s = tid; s < 256; s += 32) hw->ctBits[s] = 0;
        return;
    }
    for (unsigned s = tid; s < symbolLen; s += nthreads) {
        uint32_t c = hw->count[s];
        uint32_t r = 0;
        for (unsigned j = 0; j < symbolLen; j++) {
            uint32_t cj = hw->count[j];
            r += (cj > c) || (cj == c && j < s);
        }
        hw->ncount[1 + r] = c; hw->nsym[1 + r] = (uint8_t)s; hw->nparent[1 + r] = 0; hw->nbits[1 + r] = 0;
    }
    for (unsigned s = tid; s < 256; s += nthreads) hw->ctBits[s] = 0;
}
// Tree merge (one thread): parents of every node, nonNullRank.
B2C_DEV void huf_bt_merge(HufWork *hw) {
    uint32_t symbolLen = hw->symbolLen;
    uint32_t *cnt0 = hw->ncount;      // huffNode0
    uint32_t *cnt = hw->ncount + 1;   // huffNode
    uint16_t *par0 = hw->nparent;
    uint16_t *par = hw->nparent + 1;
    int startNode = (int)symbolLen;
    int nonNullRank = (int)symbolLen - 1;
    int nodeNb = startNode;
    while (cnt[nonNullRank] == 0) nonNullRank--;
    int lowS = nonNullRank;
    int nodeRoot = nodeNb + lowS - 1;
    int lowN = nodeNb;
    cnt[nodeNb] = cnt[lowS] + cnt[lowS - 1];
    par[lowS] = (uint16_t)nodeNb; par[lowS - 1] = (uint16_t)nodeNb;
    nodeNb++; lowS -= 2;
    for (int k = nodeNb; k <= nodeRoot; k++) cnt[k] = 1u << 30;
    cnt0[0] = 1u << 31;
    // two-queue merge; ties take the internal node (compress.go:498-519)
    uint32_t cS = cnt0[lowS + 1], cN = cnt0[lowN + 1];
    while (nodeNb <= nodeRoot) {
        int n1, n2; uint32_t c1v, c2v;
        if (cS < cN) { n1 = lowS; c1v = cS; lowS--; cS = cnt0[lowS + 1]; }
        else { n1 = lowN; c1v = cN; lowN++; cN = cnt0[lowN + 1]; }
        if (cS < cN) { n2 = lowS; c2v = cS; lowS--; cS = cnt0[lowS + 1]; }
        else { n2 = lowN; c2v = cN; lowN++; cN = cnt0[lowN + 1]; }
        uint32_t sum = c1v + c2v;
        cnt[nodeNb] = sum;
        if (lowN == nodeNb) cN = sum;  // the node just created is the head of the internal queue
        par0[n1 + 1] = (uint16_t)nodeNb; par0[n2 + 1] = (uint16_t)nodeNb;
        nodeNb++;
    }
    hw->nonNullRank = (uint32_t)nonNullRank;
}
// Depths by one warp (every lane calls): nbBits of the leaves 0..nonNullRank and of the internal nodes, by pointer
// jumping over the parent links (a node's depth doubles its reach every round: at most 8 rounds for 255 leaves).  The
// parent links are consumed (nparent holds jumped links afterwards).
B2C_DEV void huf_bt_depths(HufWork *hw, unsigned lane) {
    constexpr int PER = 16;                               // <= 510 nodes, 16 per lane
    const uint32_t startNode = hw->symbolLen, nnr = hw->nonNullRank, nodeRoot = startNode + nnr - 1;
    const uint32_t nNodes = 2 * nnr;                      // leaves 0..nnr, internal nodes startNode..nodeRoot-1
    uint16_t *par = hw->nparent + 1;
    uint8_t *nb = hw->nbits + 1;
    uint32_t pd[PER];                                     // link << 8 | distance to it
#pragma unroll
    for (int j = 0; j < PER; j++) {
        const uint32_t i = lane + 32u * (uint32_t)j;
        const uint32_t k = i <= nnr ? i : startNode + (i - nnr - 1);
        pd[j] = nodeRoot << 8 | 1u;
        if (i < nNodes) { pd[j] = (uint32_t)par[k] << 8 | 1u; nb[k] = 1; }
    }
    if (lane == 0) { par[nodeRoot] = (uint16_t)nodeRoot; nb[nodeRoot] = 0; }
    __syncwarp();
    for (;;) {
        uint32_t t[PER];
#pragma unroll
        for (int j = 0; j < PER; j++) {
            const uint32_t p = pd[j] >> 8;
            t[j] = (p != nodeRoot) ? (uint32_t)nb[p] | ((uint32_t)par[p] << 8) : 0u;
        }
        __syncwarp();
        bool more = false;
#pragma unroll
        for (int j = 0; j < PER; j++) {
            if ((pd[j] >> 8) == nodeRoot) continue;
            const uint32_t i = lane + 32u * (uint32_t)j;
            const uint32_t k = i <= nnr ? i : startNode + (i - nnr - 1);
            pd[j] = (t[j] & ~255u) | ((pd[j] & 255u) + (t[j] & 255u));   // depths stay below 256
            nb[k] = (uint8_t)pd[j]; par[k] = (uint16_t)(pd[j] >> 8);
            more |= (pd[j] >> 8) != nodeRoot;
        }
        __syncwarp();
        if (!__any_sync(FULLMASK, more)) break;
    }
}
// setMaxHeight (lane 0; it returns at once unless a code is longer than maxNbBits), then valPerRank (compress.go:536-550)
// -> scan[] for the parallel assignment, with the per-length counts from ballots.  Every lane calls.
B2C_DEV void huf_bt_ranks(HufWork *hw, uint32_t n, unsigned lane) {
    const uint32_t nnr = hw->nonNullRank;
    const uint8_t *nb = hw->nbits + 1;
    uint32_t maxNbBits = 0;
    if (lane == 0) maxNbBits = huf_set_max_height(hw, (int)nnr, huf_optimal_tablelog(11, n, hw->symbolLen));
    maxNbBits = __shfl_sync(FULLMASK, maxNbBits, 0);
    __syncwarp();
    uint32_t nbPerRank[HUF_TABLELOG_MAX + 1];
#pragma unroll
    for (int r = 0; r <= HUF_TABLELOG_MAX; r++) nbPerRank[r] = 0;
    for (uint32_t i0 = 0; i0 <= nnr; i0 += 32) {
        const uint32_t i = i0 + lane;
        const uint32_t v = i <= nnr ? nb[i] : 0u;
#pragma unroll
        for (int r = 1; r <= HUF_TABLELOG_MAX; r++) nbPerRank[r] += (uint32_t)__popc(__ballot_sync(FULLMASK, v == (uint32_t)r));
    }
    if (lane == 0) {
        hw->tableLog = maxNbBits;
        uint16_t mn = 0;
#pragma unroll
        for (int r = HUF_TABLELOG_MAX; r > 0; r--) {
            if ((uint32_t)r > maxNbBits) continue;
            hw->scan[r] = mn;
            mn = (uint16_t)(mn + nbPerRank[r]);
            mn >>= 1;
        }
    }
    __syncwarp();
}
// The whole code-length build by one warp (every lane calls).
B2C_DEV void huf_bt_tree(HufWork *hw, uint32_t n, unsigned lane) {
    if (lane == 0) huf_bt_merge(hw);
    __syncwarp();
    huf_bt_depths(hw, lane);
    huf_bt_ranks(hw, n, lane);
}
B2C_DEV void huf_bt_bits(HufWork *hw, unsigned tid, unsigned nthreads) {
    for (unsigned i = tid; i <= hw->nonNullRank; i += nthreads) hw->ctBits[hw->nsym[1 + i]] = hw->nbits[1 + i];
}
// canonical values: symbol order within each length (compress.go:552-564)
B2C_DEV void huf_bt_vals(HufWork *hw, unsigned tid, unsigned nthreads) {
    uint32_t symbolLen = hw->symbolLen;
    if (nthreads == 32) {
        // one warp: running count per code length, a ballot per length and 32 symbols
        uint32_t run[HUF_TABLELOG_MAX + 1];
#pragma unroll
        for (int b = 0; b <= HUF_TABLELOG_MAX; b++) run[b] = 0;
        for (unsigned s0 = 0; s0 < symbolLen; s0 += 32) {
            const unsigned s = s0 + tid;
            const uint32_t mb = (s < symbolLen) ? hw->ctBits[s] : 0u;
            uint32_t v = 0;
#pragma unroll
            for (int b = 1; b <= HUF_TABLELOG_MAX; b++) {
                const unsigned m = __ballot_sync(FULLMASK, mb == (uint32_t)b);
                if (mb == (uint32_t)b) v = hw->scan[b] + run[b] + (uint32_t)__popc(m & ((1u << tid) - 1));
                run[b] += (uint32_t)__popc(m);
            }
            if (s < symbolLen) hw->ctVal[s] = (uint16_t)v;
        }
        return;
    }
    for (unsigned s = tid; s < symbolLen; s += nthreads) {
        uint32_t b = hw->ctBits[s];
        uint32_t v = 0;
        if (b) {
            uint32_t before = 0;
            for (unsigned j = 0; j < s; j++) before += (hw->ctBits[j] == b);
            v = hw->scan[b] + before;
        }
        hw->ctVal[s] = (uint16_t)v;
    }
}
// cTable.write (huff0.go:180-247) by one warp (every lane calls): weights and their histogram from ballots, the FSE
// compression of huf_fse_compress_weights, or the 4-bit form.
B2C_DEV void huf_bt_write(HufWork *hw, unsigned lane) {
    const uint32_t symbolLen = hw->symbolLen;
    const uint32_t huffLog = hw->tableLog;
    const uint32_t maxSymbolValue = symbolLen - 1;
    uint32_t hist[16];
#pragma unroll
    for (int v = 0; v < 16; v++) hist[v] = 0;
    for (uint32_t k0 = 0; k0 < maxSymbolValue; k0 += 32) {
        const uint32_t k = k0 + lane;
        const bool valid = k < maxSymbolValue;
        uint32_t wv = 16;
        if (valid) {
            const uint32_t nbk = hw->ctBits[k];
            wv = nbk ? ((huffLog + 1 - nbk) & 15) : 0;
            hw->weight[k] = (uint8_t)wv;
        }
#pragma unroll
        for (int v = 0; v < 16; v++) hist[v] += (uint32_t)__popc(__ballot_sync(FULLMASK, wv == (uint32_t)v));
    }
    uint32_t *whist = hw->scan + 16;      // scan[] is free once the code values are assigned
    if (lane < 16) {
        uint32_t h = 0;
#pragma unroll
        for (int v = 0; v < 16; v++) if (lane == (unsigned)v) h = hist[v];
        whist[lane] = h;
    }
    __syncwarp();
    bool done = false;
    if (maxSymbolValue >= 2) {
        uint32_t huffMaxCnt = 0, huffMax = 0;
#pragma unroll
        for (int v = 0; v < 16; v++) {
            if (!hist[v]) continue;
            huffMax = (uint32_t)v;
            if (hist[v] > huffMaxCnt) huffMaxCnt = hist[v];
        }
        // tableDesc[0] is the size byte; the FSE payload goes to tableDesc+1..
        const int b = huf_fse_compress_weights(hw, hw->weight, maxSymbolValue, whist, huffMax + 1, huffMaxCnt,
                                               hw->tableDesc + 1, lane);
        if (b >= 0 && b < (int)(symbolLen >> 1)) {
            if (lane == 0) { hw->tableDesc[0] = (uint8_t)b; hw->tableDescLen = (uint32_t)b + 1; }
            done = true;
        }
    }
    if (!done) {
        if (maxSymbolValue > 128) { if (lane == 0) hw->status = HUF_INCOMPRESSIBLE; }
        else {
            if (lane == 0) { hw->weight[maxSymbolValue] = 0; hw->tableDesc[0] = (uint8_t)(128 | (maxSymbolValue - 1)); }
            __syncwarp();
            const uint32_t nb = (maxSymbolValue + 1) >> 1;
            for (uint32_t j = lane; j < nb; j += 32) hw->tableDesc[1 + j] = (uint8_t)((hw->weight[2 * j] << 4) | hw->weight[2 * j + 1]);
            if (lane == 0) hw->tableDescLen = 1 + nb;
        }
    }
    __syncwarp();
}
// Convenience: whole build with barriers (all threads of the group call).
// Code lengths and code values only (stages A-C): ctBits / ctVal / tableLog / symbolLen; hw->status on the early outs.
B2C_DEV void huf_build_codes(HufWork *hw, uint32_t n, unsigned tid, unsigned nthreads, int bar_id) {
#define HSYNC() do { group_sync(bar_id, (int)nthreads); } while (0)
    huf_bt_stats(hw, n, tid);
    HSYNC();
    if (hw->status != HUF_OK) return;
    huf_bt_sort(hw, tid, nthreads);
    HSYNC();
    if (tid < 32) huf_bt_tree(hw, n, tid);
    HSYNC();
    huf_bt_bits(hw, tid, nthreads);
    HSYNC();
    huf_bt_vals(hw, tid, nthreads);
    HSYNC();
#undef HSYNC
}
B2C_DEV void huf_build_table(HufWork *hw, uint32_t n, unsigned tid, unsigned nthreads, int bar_id) {
    huf_build_codes(hw, n, tid, nthreads, bar_id);
    if (hw->status != HUF_OK) return;
    if (tid < 32) huf_bt_write(hw, tid);
    group_sync(bar_id, (int)nthreads);
}

#ifndef HUF_ENC_WORDS
#define HUF_ENC_WORDS 1   // literal reads by aligned words (0: byte by byte; tuning comparison)
#endif
// ---------------------------------------------------------------- encode
// Lengths pass: every thread owns a contiguous run of symbols (in reverse order) of one of
// `nstreams` (1 or 4) segments; returns per-thread bit count; segment geometry in out params.
struct HufSeg {
    uint32_t stream;   // which stream this thread works on
    uint32_t r0, r1;   // reverse-order symbol range [r0, r1) within the stream
    uint32_t segStart; // first literal index of the stream
    uint32_t segLen;   // symbols in the stream
};
B2C_DEV HufSeg huf_thread_seg(uint32_t n, int nstreams, unsigned tid, unsigned nthreads) {
    HufSeg s;
    unsigned per = nthreads / (unsigned)nstreams;  // threads per stream
    s.stream = tid / per;
    unsigned t = tid % per;
    uint32_t segmentSize = (nstreams == 4) ? (n + 3) / 4 : n;
    s.segStart = s.stream * segmentSize;
    uint32_t end = s.segStart + segmentSize;
    if (end > n) end = n;
    s.segLen = (s.segStart < n) ? end - s.segStart : 0;
    uint32_t chunk = (s.segLen + per - 1) / per;
    s.r0 = t * chunk; if (s.r0 > s.segLen) s.r0 = s.segLen;
    s.r1 = s.r0 + chunk; if (s.r1 > s.segLen) s.r1 = s.segLen;
    return s;
}

// Encoding is split in two collective calls so the caller can size headers in between:
//   huf_enc_sizes : per-thread code-length sums + block scan -> stream sizes, total payload bytes
//   huf_enc_pack  : every thread packs its bit range into the zeroed staging words
struct HufEncState {
    HufSeg sg;
    uint32_t myoff;   // bit offset of my run inside my stream
    uint32_t soff;    // byte offset of my stream inside the payload
    uint32_t t;       // thread index inside the stream group
};
// returns payload bytes = table desc + (jump table) + streams
// pk: 256 words of caller-provided shared scratch; filled here with (code | nbits << 16) for huf_enc_pack.
B2C_DEV uint32_t huf_enc_sizes(HufWork *hw, uint32_t *pk, const uint8_t *lit, uint32_t n, int four, unsigned tid,
                               unsigned nthreads, int bar_id, HufEncState *st) {
#define HSYNC() do { group_sync(bar_id, (int)nthreads); } while (0)
    int nstreams = four ? 4 : 1;
    HufSeg sg = huf_thread_seg(n, nstreams, tid, nthreads);
    unsigned per = nthreads / (unsigned)nstreams;
    unsigned t = tid % per;
    for (unsigned s = tid; s < 256; s += nthreads) pk[s] = (uint32_t)hw->ctVal[s] | ((uint32_t)hw->ctBits[s] << 16);
    uint32_t mybits = 0;
    {
        // my symbols are the bytes [a, b) of lit; the sum does not depend on the order: aligned words in the middle
        const uint8_t *cb = hw->ctBits;
        uint32_t i = sg.segStart + sg.segLen - sg.r1;
        const uint32_t b = sg.segStart + sg.segLen - sg.r0;
        while (i < b && (reinterpret_cast<uintptr_t>(lit + i) & 3)) mybits += cb[lit[i++]];
        for (; HUF_ENC_WORDS && i + 4 <= b; i += 4) {
            const uint32_t w = *reinterpret_cast<const uint32_t *>(lit + i);
            mybits += (uint32_t)cb[w & 255] + cb[(w >> 8) & 255] + cb[(w >> 16) & 255] + cb[w >> 24];
        }
        while (i < b) mybits += cb[lit[i++]];
    }
    uint32_t total;
    uint32_t ex = group_scan_excl(mybits, hw->scan, bar_id, (int)nthreads, tid, &total);
    if (t == 0) hw->streamBits[sg.stream] = ex;  // temporarily: the stream's base in the global scan
    HSYNC();
    uint32_t base = hw->streamBits[sg.stream];
    uint32_t nextBase = (sg.stream + 1 < (uint32_t)nstreams) ? hw->streamBits[sg.stream + 1] : total;
    uint32_t sbits = nextBase - base;
    HSYNC();
    if (t == 0) { hw->streamBits[sg.stream] = sbits; hw->streamBytes[sg.stream] = (sbits + 1 + 7) >> 3; }
    HSYNC();
    uint32_t hdr = hw->tableDescLen + (four ? 6u : 0u);
    uint32_t soff = hdr;
    for (uint32_t k = 0; k < sg.stream; k++) soff += hw->streamBytes[k];
    uint32_t totalBytes = hdr;
    for (int k = 0; k < nstreams; k++) totalBytes += hw->streamBytes[k];
    st->sg = sg; st->myoff = ex - base; st->soff = soff; st->t = t;
#undef HSYNC
    return totalBytes;
}
// The two halves of huf_enc_pack, for callers that order them against their own stores:
//   huf_enc_pack_bits   : the streams, word-granular (plain stores and atomicOr into the zeroed staging words)
//   huf_enc_pack_header : the table description and the jump table, byte stores; a barrier must separate the two.
B2C_DEV void huf_enc_pack_bits(const uint32_t *pk, const uint8_t *lit, uint8_t *stageBase, uint32_t byteOff,
                               const HufEncState *st) {
    const HufSeg &sg = st->sg;
    {
        BitRun br;
        br.init(reinterpret_cast<uint32_t *>(stageBase), (byteOff + st->soff) * 8 + st->myoff);
        // bytes [a, b) of lit, emitted from b-1 down to a; codes are <= 11 bits, so two go into one add
        const uint32_t a = sg.segStart + sg.segLen - sg.r1;
        uint32_t i = sg.segStart + sg.segLen - sg.r0;
        while (i > a && (reinterpret_cast<uintptr_t>(lit + i) & 3)) {
            const uint32_t e = pk[lit[--i]];
            br.add(e & 0xffffu, e >> 16);
        }
        for (; HUF_ENC_WORDS && i >= a + 4; i -= 4) {
            const uint32_t w = *reinterpret_cast<const uint32_t *>(lit + i - 4);
            const uint32_t e3 = pk[w >> 24], e2 = pk[(w >> 16) & 255], e1 = pk[(w >> 8) & 255], e0 = pk[w & 255];
            br.add((e3 & 0xffffu) | ((e2 & 0xffffu) << (e3 >> 16)), (e3 >> 16) + (e2 >> 16));
            br.add((e1 & 0xffffu) | ((e0 & 0xffffu) << (e1 >> 16)), (e1 >> 16) + (e0 >> 16));
        }
        while (i > a) {
            const uint32_t e = pk[lit[--i]];
            br.add(e & 0xffffu, e >> 16);
        }
        // end mark: added by the thread that owns the last symbol (or thread 0 of an empty stream)
        bool last = (sg.segLen == 0) ? (st->t == 0) : (sg.r1 == sg.segLen && sg.r0 < sg.r1);
        if (last) br.add(1u, 1);
        br.finish();
    }
}
B2C_DEV void huf_enc_pack_header(const HufWork *hw, int four, uint8_t *stageBase, uint32_t byteOff, unsigned tid,
                                 unsigned nthreads) {
    uint8_t *stage = stageBase + byteOff;
    for (unsigned i = tid; i < hw->tableDescLen; i += nthreads) stage[i] = hw->tableDesc[i];
    if (four && tid < 3) {
        uint32_t L = hw->streamBytes[tid];
        stage[hw->tableDescLen + tid * 2] = (uint8_t)L;
        stage[hw->tableDescLen + tid * 2 + 1] = (uint8_t)(L >> 8);
    }
}
// stageBase: 4-byte aligned, zero-initialised words; payload starts at byte offset byteOff.
// pk: the table huf_enc_sizes filled (a barrier lies between the two calls).
B2C_DEV void huf_enc_pack(HufWork *hw, const uint32_t *pk, const uint8_t *lit, int four, uint8_t *stageBase,
                          uint32_t byteOff, unsigned tid, unsigned nthreads, int bar_id, const HufEncState *st) {
    huf_enc_pack_bits(pk, lit, stageBase, byteOff, st);
    group_sync(bar_id, (int)nthreads);
    // header bytes (byte stores, ordered after the word-granular atomics above)
    huf_enc_pack_header(hw, four, stageBase, byteOff, tid, nthreads);
    group_sync(bar_id, (int)nthreads);
}

}  // namespace b2c
