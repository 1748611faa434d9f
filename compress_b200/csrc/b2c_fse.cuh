// compress_b200/csrc/b2c_fse.cuh -- FSE (tANS) table construction on the device.
//
// Replaces, for the GPU path, the reference's
//   zstd/fse_encoder.go:102-204 (buildCTable), :259-427 (normalizeCount/2),
//   :429-455 (optimalTableLog), :488-598 (writeCount), :603-672 (bitCost/approxSize)
//   fse/compress.go (same arithmetic, used for huff0 weight tables).
// Tables here are tiny (<= 64 symbols, <= 256 states); each table is built by one
// warp (normalisation, table fill and size estimates over its lanes; the NCount and
// the predefined tables on one thread).  All results are bit-exact with the oracle.
#pragma once
#include "b2c_common.cuh"

namespace b2c {

constexpr int FSE_MAX_SYM = 64;
constexpr int FSE_MAX_STATES = 256;

struct FseCTable {
    uint16_t stateTable[FSE_MAX_STATES];
    uint8_t tableSymbol[FSE_MAX_STATES];
    uint32_t deltaNbBits[FSE_MAX_SYM];
    int16_t deltaFindState[FSE_MAX_SYM];
    int16_t norm[FSE_MAX_SYM];
    uint32_t symbolLen;
    uint32_t tableLog;
    uint32_t useRLE;
    uint32_t rleVal;
};

B2C_DEV uint32_t fse_hb(uint32_t v) { return v ? highbit32(v) : 0xffffffffu; }  // Go bits.Len32(v)-1

// normalizeCount2 (secondary method)
B2C_DEV int fse_normalize2(const uint32_t *count, uint32_t symbolLen, uint32_t length, uint32_t tableLog,
                           int16_t *norm) {
    const int16_t notYetAssigned = -2;
    uint32_t distributed = 0, total = length;
    uint32_t lowThreshold = total >> tableLog;
    uint32_t lowOne = (total * 3) >> (tableLog + 1);
    for (uint32_t i = 0; i < symbolLen; i++) {
        uint32_t cnt = count[i];
        if (cnt == 0) { norm[i] = 0; continue; }
        if (cnt <= lowThreshold) { norm[i] = -1; distributed++; total -= cnt; continue; }
        if (cnt <= lowOne) { norm[i] = 1; distributed++; total -= cnt; continue; }
        norm[i] = notYetAssigned;
    }
    uint32_t toDistribute = (1u << tableLog) - distributed;
    if ((total / toDistribute) > lowOne) {
        lowOne = (total * 3) / (toDistribute * 2);
        for (uint32_t i = 0; i < symbolLen; i++) {
            if (norm[i] == notYetAssigned && count[i] <= lowOne) { norm[i] = 1; distributed++; total -= count[i]; }
        }
        toDistribute = (1u << tableLog) - distributed;
    }
    if (distributed == symbolLen + 1) {
        uint32_t maxV = 0, maxC = 0;
        for (uint32_t i = 0; i < symbolLen; i++) if (count[i] > maxC) { maxV = i; maxC = count[i]; }
        norm[maxV] = (int16_t)(norm[maxV] + (int16_t)toDistribute);
        return 0;
    }
    if (total == 0) {
        for (uint32_t i = 0; toDistribute > 0; i = (i + 1) % symbolLen) {
            if (norm[i] > 0) { toDistribute--; norm[i]++; }
        }
        return 0;
    }
    uint64_t vStepLog = 62 - (uint64_t)tableLog;
    uint64_t mid = (1ull << (vStepLog - 1)) - 1;
    uint64_t rStep = (((1ull << vStepLog) * (uint64_t)toDistribute) + mid) / (uint64_t)total;
    uint64_t tmpTotal = mid;
    for (uint32_t i = 0; i < symbolLen; i++) {
        if (norm[i] == notYetAssigned) {
            uint64_t end = tmpTotal + (uint64_t)count[i] * rStep;
            uint32_t sStart = (uint32_t)(tmpTotal >> vStepLog);
            uint32_t sEnd = (uint32_t)(end >> vStepLog);
            uint32_t weight = sEnd - sStart;
            if (weight < 1) return -1;
            norm[i] = (int16_t)weight;
            tmpTotal = end;
        }
    }
    return 0;
}

// normalizeCount by one warp (symbolLen <= 64: symbols lane and lane + 32); every lane calls and gets the same result.
// The serial loop's running largest (first symbol with the highest probability) is a warp arg-max with the same tie
// rule; the rare fall-back to normalizeCount2 runs on lane 0.
B2C_DEV int fse_normalize(const uint32_t *count, uint32_t symbolLen, uint32_t length, uint32_t tableLog,
                          int16_t *norm, unsigned lane) {
    const uint32_t rtb[8] = {0, 473195, 504333, 520860, 550000, 700000, 750000, 830000};
    const uint64_t scale = 62 - (uint64_t)tableLog;
    const uint64_t step = (1ull << 62) / (uint64_t)length;
    const uint64_t vStep = 1ull << (scale - 20);
    const uint32_t lowThreshold = length >> tableLog;
    int used = 0;           // states this lane's symbols take
    uint32_t key = 0;       // proba << 8 | (255 - symbol) of this lane's best symbol (0: none)
#pragma unroll
    for (int h = 0; h < 2; h++) {
        const uint32_t i = lane + 32u * (uint32_t)h;
        if (i >= symbolLen) continue;
        const uint32_t cnt = count[i];
        int proba = 0;
        if (cnt == 0) proba = 0;
        else if (cnt <= lowThreshold) { proba = -1; used += 1; }
        else {
            proba = (int)(((uint64_t)cnt * step) >> scale);
            if (proba < 8) {
                const uint64_t restToBeat = vStep * (uint64_t)rtb[proba];
                const uint64_t v = (uint64_t)cnt * step - ((uint64_t)proba << scale);
                if (v > restToBeat) proba++;
            }
            used += proba;
            const uint32_t k = ((uint32_t)proba << 8) | (255u - i);
            if (proba > 0 && k > key) key = k;
        }
        norm[i] = (int16_t)proba;
    }
    const int stillToDistribute = (1 << tableLog) - (int)warp_sum((uint32_t)used);
    key = warp_max(key);
    const uint32_t largest = key ? 255u - (key & 255u) : 0u;
    __syncwarp();
    const int largestP = key ? (int)(key >> 8) : (int)norm[0];   // norm[largest]
    if (-stillToDistribute >= (largestP >> 1)) {
        int r = 0;
        if (lane == 0) r = fse_normalize2(count, symbolLen, length, tableLog, norm);
        r = __shfl_sync(FULLMASK, r, 0);
        __syncwarp();
        return r;
    }
    if (lane == 0) norm[largest] = (int16_t)(largestP + stillToDistribute);
    __syncwarp();
    return 0;
}

// writeCount: returns bytes written (out must have 2 bytes of slack), <0 on internal error
B2C_DEV int fse_write_ncount(const int16_t *norm, uint32_t symbolLen, uint32_t tableLog, uint8_t *out) {
    int tableSize = 1 << tableLog;
    bool previous0 = false;
    uint32_t charnum = 0;
    uint32_t bitStream = tableLog - 5;
    uint32_t bitCount = 4;
    int16_t remaining = (int16_t)(tableSize + 1);
    int16_t threshold = (int16_t)tableSize;
    uint32_t nbBits = tableLog + 1;
    uint32_t outP = 0;
    while (remaining > 1) {
        if (previous0) {
            uint32_t start = charnum;
            while (norm[charnum] == 0) charnum++;
            while (charnum >= start + 24) {
                start += 24;
                bitStream += 0xFFFFu << bitCount;
                out[outP] = (uint8_t)bitStream; out[outP + 1] = (uint8_t)(bitStream >> 8); outP += 2;
                bitStream >>= 16;
            }
            while (charnum >= start + 3) { start += 3; bitStream += 3u << bitCount; bitCount += 2; }
            bitStream += (charnum - start) << bitCount;
            bitCount += 2;
            if (bitCount > 16) {
                out[outP] = (uint8_t)bitStream; out[outP + 1] = (uint8_t)(bitStream >> 8); outP += 2;
                bitStream >>= 16; bitCount -= 16;
            }
        }
        int16_t count = norm[charnum];
        charnum++;
        int16_t max = (int16_t)((2 * threshold - 1) - remaining);
        if (count < 0) remaining = (int16_t)(remaining + count);
        else remaining = (int16_t)(remaining - count);
        count++;
        if (count >= threshold) count = (int16_t)(count + max);
        bitStream += (uint32_t)count << bitCount;
        bitCount += nbBits;
        if (count < max) bitCount--;
        previous0 = (count == 1);
        if (remaining < 1) return -1;
        while (remaining < threshold) { nbBits--; threshold >>= 1; }
        if (bitCount > 16) {
            out[outP] = (uint8_t)bitStream; out[outP + 1] = (uint8_t)(bitStream >> 8); outP += 2;
            bitStream >>= 16; bitCount -= 16;
        }
    }
    out[outP] = (uint8_t)bitStream;
    out[outP + 1] = (uint8_t)(bitStream >> 8);
    outP += (bitCount + 7) / 8;
    if (charnum > symbolLen) return -1;
    return (int)outP;
}

// buildCTable from ct->norm / symbolLen / tableLog
B2C_DEV int fse_build_ctable(FseCTable *ct) {
    const int16_t *norm = ct->norm;
    uint32_t symbolLen = ct->symbolLen, tableLog = ct->tableLog;
    uint32_t tableSize = 1u << tableLog;
    uint32_t highThreshold = tableSize - 1;
    int16_t cumul[FSE_MAX_SYM + 2];
    cumul[0] = 0;
    for (uint32_t u = 0; u < symbolLen; u++) {
        int16_t v = norm[u];
        if (v == -1) {
            cumul[u + 1] = (int16_t)(cumul[u] + 1);
            ct->tableSymbol[highThreshold] = (uint8_t)u;
            highThreshold--;
        } else {
            cumul[u + 1] = (int16_t)(cumul[u] + v);
        }
    }
    if ((uint32_t)cumul[symbolLen] != tableSize) return -1;
    cumul[symbolLen] = (int16_t)(tableSize + 1);
    {
        uint32_t step = (tableSize >> 1) + (tableSize >> 3) + 3;
        uint32_t tableMask = tableSize - 1;
        uint32_t position = 0;
        for (uint32_t ui = 0; ui < symbolLen; ui++) {
            int v = norm[ui];
            for (int n = 0; n < v; n++) {
                ct->tableSymbol[position] = (uint8_t)ui;
                position = (position + step) & tableMask;
                while (position > highThreshold) position = (position + step) & tableMask;
            }
        }
        if (position != 0) return -1;
    }
    for (uint32_t u = 0; u < tableSize; u++) {
        uint8_t v = ct->tableSymbol[u];
        ct->stateTable[cumul[v]] = (uint16_t)(tableSize + u);
        cumul[v]++;
    }
    {
        int16_t total = 0;
        uint32_t tl = (tableLog << 16) - (1u << tableLog);
        for (uint32_t i = 0; i < symbolLen; i++) {
            int16_t v = norm[i];
            if (v == 0) { ct->deltaNbBits[i] = 0; ct->deltaFindState[i] = 0; continue; }
            if (v == -1 || v == 1) {
                ct->deltaNbBits[i] = tl;
                ct->deltaFindState[i] = (int16_t)(total - 1);
                total++;
            } else {
                uint32_t maxBitsOut = tableLog - highbit32((uint32_t)(v - 1));
                uint32_t minStatePlus = (uint32_t)v << maxBitsOut;
                ct->deltaNbBits[i] = (maxBitsOut << 16) - minStatePlus;
                ct->deltaFindState[i] = (int16_t)(total - v);
                total = (int16_t)(total + v);
            }
        }
        if (total != (int16_t)tableSize) return -1;
    }
    return 0;
}

// buildCTable by one warp (ct in shared memory; scratch: 3 * 66 uint16 of shared memory).  Same table as
// fse_build_ctable (fse_encoder.go:102-203); the serial symbol spread and state fill are replaced by rank computations:
//   cell order k -> position (k * step) & mask, skipped when above highThreshold; the j-th surviving cell receives the
//   symbol whose cumulative positive count covers j; state slot of cell u = cumul[symbol] + #(earlier cells, same symbol).
B2C_DEV int fse_build_ctable_warp(FseCTable *ct, uint16_t *scratch, unsigned lane) {
    const int16_t *norm = ct->norm;
    const uint32_t symbolLen = ct->symbolLen, tableLog = ct->tableLog, tableSize = 1u << tableLog;
    uint16_t *cumul = scratch;          // [65] counts with -1 taken as 1
    uint16_t *cpos = scratch + 66;      // [65] positive counts only
    uint16_t *fill = scratch + 132;     // [64] running per-symbol fill counters
    // ---- cumulative counts (two symbols per lane)
    const uint32_t i0 = lane, i1 = lane + 32;
    const int v0 = (i0 < symbolLen) ? norm[i0] : 0, v1 = (i1 < symbolLen) ? norm[i1] : 0;
    const uint32_t a0 = v0 == -1 ? 1u : (uint32_t)v0, a1 = v1 == -1 ? 1u : (uint32_t)v1;
    const uint32_t p0 = v0 > 0 ? (uint32_t)v0 : 0u, p1 = v1 > 0 ? (uint32_t)v1 : 0u;
    const uint32_t packed0 = a0 | (p0 << 16), packed1 = a1 | (p1 << 16);
    const uint32_t inc0 = warp_scan_incl(packed0);
    const uint32_t tot0 = __shfl_sync(FULLMASK, inc0, 31);
    const uint32_t inc1 = warp_scan_incl(packed1) + tot0;
    const uint32_t ex0 = inc0 - packed0, ex1 = inc1 - packed1;
    cumul[i0] = (uint16_t)ex0; cumul[i1] = (uint16_t)ex1;
    cpos[i0] = (uint16_t)(ex0 >> 16); cpos[i1] = (uint16_t)(ex1 >> 16);
    fill[i0] = 0; fill[i1] = 0;
    const uint32_t grand = __shfl_sync(FULLMASK, inc1, 31);
    if (lane == 31) { cumul[64] = (uint16_t)grand; cpos[64] = (uint16_t)(grand >> 16); }
    if ((grand & 0xffff) != tableSize) return -1;
    const uint32_t nPos = grand >> 16;            // cells filled by the spread
    // low-probability symbols take the top cells, lowest symbol highest
    const unsigned m0 = __ballot_sync(FULLMASK, v0 == -1), m1 = __ballot_sync(FULLMASK, v1 == -1);
    const uint32_t nLow0 = (uint32_t)__popc(m0), nLow = nLow0 + (uint32_t)__popc(m1);
    if (v0 == -1) ct->tableSymbol[tableSize - 1 - (uint32_t)__popc(m0 & ((1u << lane) - 1))] = (uint8_t)i0;
    if (v1 == -1) ct->tableSymbol[tableSize - 1 - nLow0 - (uint32_t)__popc(m1 & ((1u << lane) - 1))] = (uint8_t)i1;
    const uint32_t highThreshold = tableSize - 1 - nLow;
    __syncwarp();
    // ---- spread
    {
        const uint32_t step = (tableSize >> 1) + (tableSize >> 3) + 3, tableMask = tableSize - 1;
        uint32_t base = 0;
        for (uint32_t k0 = 0; k0 < tableSize; k0 += 32) {
            const uint32_t k = k0 + lane;
            const uint32_t pos = (k * step) & tableMask;
            const bool ok = (k < tableSize) && (pos <= highThreshold);
            const unsigned okm = __ballot_sync(FULLMASK, ok);
            if (ok) {
                const uint32_t j = base + (uint32_t)__popc(okm & ((1u << lane) - 1));
                // largest s with cpos[s] <= j (symbols with no cells share the value of their successor and are skipped)
                uint32_t lo = 0, hi = symbolLen;         // invariant: cpos[lo] <= j < cpos[hi]
                while (hi - lo > 1) {
                    const uint32_t mid = (lo + hi) >> 1;
                    if (cpos[mid] <= j) lo = mid; else hi = mid;
                }
                ct->tableSymbol[pos] = (uint8_t)lo;
            }
            base += (uint32_t)__popc(okm);
        }
        if (base != nPos) return -1;
    }
    __syncwarp();
    // ---- state table: cells in position order
    for (uint32_t u0 = 0; u0 < tableSize; u0 += 32) {
        const uint32_t u = u0 + lane;
        const bool ok = u < tableSize;
        const unsigned okm = __ballot_sync(FULLMASK, ok);
        if (ok) {
            const uint32_t sym = ct->tableSymbol[u];
            const unsigned peers = __match_any_sync(okm, sym);
            const uint32_t before = fill[sym];
            __syncwarp(okm);
            ct->stateTable[cumul[sym] + before + (uint32_t)__popc(peers & ((1u << lane) - 1))] = (uint16_t)(tableSize + u);
            if (lane == (unsigned)(__ffs((int)peers) - 1)) fill[sym] = (uint16_t)(before + (uint32_t)__popc(peers));
        }
        __syncwarp();
    }
    // ---- symbol transforms
    {
        const uint32_t tl = (tableLog << 16) - (1u << tableLog);
        for (uint32_t i = lane; i < symbolLen; i += 32) {
            const int v = norm[i];
            if (v == 0) { ct->deltaNbBits[i] = 0; ct->deltaFindState[i] = 0; }
            else if (v == -1 || v == 1) { ct->deltaNbBits[i] = tl; ct->deltaFindState[i] = (int16_t)((int)cumul[i] - 1); }
            else {
                const uint32_t maxBitsOut = tableLog - highbit32((uint32_t)(v - 1));
                const uint32_t minStatePlus = (uint32_t)v << maxBitsOut;
                ct->deltaNbBits[i] = (maxBitsOut << 16) - minStatePlus;
                ct->deltaFindState[i] = (int16_t)((int)cumul[i] - v);
            }
        }
    }
    __syncwarp();
    return 0;
}

// cState.init
B2C_DEV uint32_t fse_init_state(const FseCTable *ct, uint32_t sym) {
    if (ct->useRLE) return 0;
    uint32_t dnb = ct->deltaNbBits[sym];
    uint32_t nbBitsOut = (dnb + (1u << 15)) >> 16;
    int32_t im = (int32_t)((nbBitsOut << 16) - dnb);
    int32_t lu = (im >> nbBitsOut) + (int32_t)ct->deltaFindState[sym];
    return ct->stateTable[lu];
}

// bitCost / approxSize (hist length = histLen <= 64) by one warp: symbols lane and lane + 32, a warp sum (the 32-bit
// sum wraps the same in any order).  Every lane calls and gets the same result.
B2C_DEV uint32_t fse_approx_size(const FseCTable *s, const uint32_t *hist, uint32_t histLen, unsigned lane) {
    if (s->symbolLen < histLen) return 0xffffffffu;
    if (s->useRLE) return 0xffffffffu;
    const uint32_t kAcc = 8;
    const uint32_t badCost = (s->tableLog + 1) << kAcc;
    uint32_t cost = 0;
    bool bad = false;
#pragma unroll
    for (int h = 0; h < 2; h++) {
        const uint32_t i = lane + 32u * (uint32_t)h;
        if (i >= histLen || hist[i] == 0) continue;
        if (s->norm[i] == 0) { bad = true; continue; }
        const uint32_t dnb = s->deltaNbBits[i];
        const uint32_t minNbBits = dnb >> 16;
        const uint32_t threshold = (minNbBits + 1) << 16;
        const uint32_t tableSize = 1u << s->tableLog;
        const uint32_t deltaFromThreshold = threshold - (dnb + tableSize);
        const uint32_t normalizedDelta = (deltaFromThreshold << kAcc) >> s->tableLog;
        const uint32_t bc = (minNbBits + 1) * (1u << kAcc) - normalizedDelta;
        if (bc > badCost) { bad = true; continue; }
        cost += hist[i] * bc;
    }
    if (__any_sync(FULLMASK, bad)) return 0xffffffffu;
    return warp_sum(cost) >> kAcc;
}

}  // namespace b2c
