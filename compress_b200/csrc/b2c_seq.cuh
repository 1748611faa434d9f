// compress_b200/csrc/b2c_seq.cuh -- zstd sequence section on the device.
//
// Device-native replacement for the reference's
//   zstd/blockenc.go:601-610 (nSeq header), :611-724 (modes, chooseComp, NCount tables),
//   :725-808 (3-state backward FSE bitstream), :831-893 (genCodes)
//   zstd/seqenc.go:48-112 (llCode/mlCode/ofCode + extra-bit tables)
//   zstd/fse_encoder.go (normalizeCount/buildCTable/writeCount/approxSize, via b2c_fse.cuh)
//   zstd/fse_predefined.go:118-156 (default distributions)
// Code tables, the predefined tables and the per-block table build (K2); the state chains themselves are walked by
// zstd_chains_block (b2c_zstd_enc.cuh).  Output bytes equal the oracle's.
#pragma once
#include "b2c_common.cuh"
#include "b2c_fse.cuh"

namespace b2c {

enum { TBL_LL = 0, TBL_OF = 1, TBL_ML = 2 };
constexpr uint32_t SEQ_TABLE_ERR = 0xffffffffu;  // ncountLen marker: table construction failed

// The predefined tables (fse_predefined.go), built once per CTA and read by every warp's mode decision.
struct SeqWork {
    FseCTable predef[3];
};
// One warp's scratch for building one sequence table.
struct SeqTableWork {
    FseCTable cur;
    uint32_t hist[64];
    uint32_t mode;             // 0 predefined, 1 RLE, 2 FSE
    uint32_t used;             // 0 -> the predefined table, 1 -> cur
    uint32_t ncountLen;
    uint8_t ncount[96];
    uint16_t fseScratch[200];  // fse_build_ctable_warp
};

B2C_DEV uint32_t seq_ll_code(uint32_t litLength) {
    // seqenc.go:48-75
    if (litLength <= 15) return litLength;
    if (litLength <= 63) {
        if (litLength < 24) return 16 + ((litLength - 16) >> 1);
        if (litLength < 32) return 20 + ((litLength - 24) >> 2);
        if (litLength < 40) return 22;
        if (litLength < 48) return 23;
        return 24;
    }
    return highbit32(litLength) + 19;
}
B2C_DEV uint32_t seq_ml_code(uint32_t mlBase) {
    // seqenc.go:77-107
    if (mlBase <= 31) return mlBase;
    if (mlBase <= 127) {
        if (mlBase < 40) return 32 + ((mlBase - 32) >> 1);
        if (mlBase < 48) return 36 + ((mlBase - 40) >> 2);
        if (mlBase < 56) return 38;
        if (mlBase < 64) return 39;
        if (mlBase < 80) return 40;
        if (mlBase < 96) return 41;
        return 42;
    }
    return highbit32(mlBase) + 36;
}
B2C_DEV uint32_t seq_ll_bits(uint32_t code) {  // llBitsTable, seqenc.go:61-66
    if (code < 16) return 0;
    if (code < 20) return 1;
    if (code < 22) return 2;
    if (code < 24) return 3;
    if (code == 24) return 4;
    return code - 19;  // 25 -> 6, 26 -> 7 ... 35 -> 16
}
B2C_DEV uint32_t seq_ml_bits(uint32_t code) {  // mlBitsTable, seqenc.go:90-97
    if (code < 32) return 0;
    if (code < 36) return 1;
    if (code < 38) return 2;
    if (code < 40) return 3;
    if (code < 42) return 4;
    if (code == 42) return 5;
    return code - 36;  // 43 -> 7 ... 52 -> 16
}

// Build the three predefined encoder tables (one thread each; tid 0..2 of the caller's choice).
B2C_DEV void seq_build_predef(SeqWork *sw, int which) {
    const int8_t llN[36] = {4, 3, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 1, 1, 1, 2, 2,
                            2, 2, 2, 2, 2, 2, 2, 3, 2, 1, 1, 1, 1, 1, -1, -1, -1, -1};
    const int8_t ofN[29] = {1, 1, 1, 1, 1, 1, 2, 2, 2, 1, 1, 1, 1, 1, 1,
                            1, 1, 1, 1, 1, 1, 1, 1, 1, -1, -1, -1, -1, -1};
    const int8_t mlN[53] = {1, 4, 3, 2, 2, 2, 2, 2, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1,
                            1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1,
                            1, 1, 1, 1, 1, 1, 1, 1, 1, 1, -1, -1, -1, -1, -1, -1, -1};
    FseCTable *ct = &sw->predef[which];
    for (int i = 0; i < FSE_MAX_SYM; i++) ct->norm[i] = 0;
    if (which == TBL_LL) { for (int i = 0; i < 36; i++) ct->norm[i] = llN[i]; ct->symbolLen = 36; ct->tableLog = 6; }
    else if (which == TBL_OF) { for (int i = 0; i < 29; i++) ct->norm[i] = ofN[i]; ct->symbolLen = 29; ct->tableLog = 5; }
    else { for (int i = 0; i < 53; i++) ct->norm[i] = mlN[i]; ct->symbolLen = 53; ct->tableLog = 6; }
    ct->useRLE = 0; ct->rleVal = 0;
    fse_build_ctable(ct);
}

// fseEncoder.optimalTableLog (fse_encoder.go:429-455)
B2C_DEV uint32_t seq_optimal_tablelog(uint32_t length, uint32_t symbolLen) {
    uint8_t tableLog = 8;
    uint32_t minBitsSrc = fse_hb(length) + 1;
    uint32_t minBitsSymbols = fse_hb(symbolLen - 1) + 2;
    uint8_t minBits = (uint8_t)minBitsSymbols;
    if (minBitsSrc < minBitsSymbols) minBits = (uint8_t)minBitsSrc;
    uint8_t maxBitsSrc = (uint8_t)((uint8_t)fse_hb(length - 1) - 2);
    if (maxBitsSrc < tableLog) tableLog = maxBitsSrc;
    if (minBits > tableLog) tableLog = minBits;
    if (tableLog < 5) tableLog = 5;
    if (tableLog > 8) tableLog = 8;
    return tableLog;
}

// One warp builds a table from st->hist (fresh block: no previous tables); every lane calls.  predef: the predefined table
// of the same kind.  firstCode = code of sequence 0 (setRLE uses b.sequences[0]).  Normalisation, table fill and size
// estimates use all lanes; the NCount is written by lane 0.
// row: optional profiling stamps (stamp_clock) 0 start, 1 normalised, 2 table filled, 3 sizes estimated, 4 NCount written.
B2C_DEV void seq_build_table(SeqTableWork *st, const FseCTable *predef, uint32_t symbolLen, uint32_t nseq,
                             uint32_t firstCode, unsigned lane, unsigned long long *row) {
    stamp_clock(row, 0);
    FseCTable *ct = &st->cur;
    const uint32_t *hist = st->hist;
    uint32_t maxCount = warp_max(hist[lane] > hist[lane + 32] ? hist[lane] : hist[lane + 32]);   // bins >= symbolLen are zero
    const uint32_t tableLog = seq_optimal_tablelog(nseq, symbolLen);
    if (lane == 0) {
        ct->symbolLen = symbolLen;
        ct->tableLog = tableLog;
        ct->rleVal = 0;
    }
    if (maxCount == nseq) {
        // useRLE: setRLE(b.sequences[0].code), fse_encoder.go:208-221
        if (lane == 0) {
            ct->useRLE = 1; ct->rleVal = firstCode; ct->tableLog = 0;
            ct->stateTable[0] = 0; ct->deltaNbBits[firstCode] = 0; ct->deltaFindState[firstCode] = 0;
            st->mode = 1; st->used = 1;
            st->ncount[0] = (uint8_t)firstCode; st->ncountLen = 1;
        }
        __syncwarp();
        return;
    }
    ct->norm[lane] = 0; ct->norm[lane + 32] = 0;
    if (lane == 0) ct->useRLE = 0;
    __syncwarp();
    int bad = fse_normalize(hist, symbolLen, nseq, tableLog, ct->norm, lane);
    stamp_clock(row, 1);
    if (!bad) bad = fse_build_ctable_warp(ct, st->fseScratch, lane);
    stamp_clock(row, 2);
    if (bad) {
        if (lane == 0) { st->mode = 0; st->used = 0; st->ncountLen = SEQ_TABLE_ERR; }
        __syncwarp();
        return;
    }
    // chooseComp, blockenc.go:633-661 (prev == never valid for an independent block)
    uint32_t nSize = fse_approx_size(ct, hist, symbolLen, lane) + (((symbolLen * tableLog) >> 3) + 3) * 8;
    const uint32_t predefSize = fse_approx_size(predef, hist, symbolLen, lane);
    nSize = nSize + ((nSize + 2 * 8 * 16) >> 4);
    stamp_clock(row, 3);
    if (lane == 0) {
        if (predefSize <= nSize) { st->mode = 0; st->used = 0; st->ncountLen = 0; }
        else {
            st->mode = 2; st->used = 1;
            int w = fse_write_ncount(ct->norm, symbolLen, tableLog, st->ncount);
            if (w < 0) { st->mode = 0; st->used = 0; st->ncountLen = SEQ_TABLE_ERR; }
            else st->ncountLen = (uint32_t)w;
        }
        stamp_clock(row, 4);
    }
    __syncwarp();
}

}  // namespace b2c
