// tests/emu/emu_lz4.cpp -- the LZ4 / LZ4s -> S2 / Snappy conversion kernels (b2c_lz4_cvt.cuh) under the SIMT emulator.
// TEST INFRASTRUCTURE ONLY.
#include "simt_emu.h"
#include "../../compress_b200/csrc/b2c_lz4_cvt.cuh"
#include <vector>

using namespace b2c;

extern "C" {

void emu_lz4_set_lane_order(int desc) { emu::lane_order_desc = desc; }

// The device's two kernels: walk (one lane per block), emit (one warp per block).  Blocks at src + src_off[i]
// (src_sizes[i] bytes), slots at dst + dst_off[i] (dst_caps[i] bytes); the host call's record layout.
int emu_lz4_convert(const uint8_t *src, const uint64_t *src_off, const uint32_t *src_sizes, uint32_t n, uint8_t *dst,
                    const uint64_t *dst_off, const uint32_t *dst_caps, int64_t *out_sizes, int64_t *decoded, int lz4s, int snappy) {
    LzcParams P;
    memset(&P, 0, sizeof(P));
    P.src_base = src; P.src_offsets = src_off; P.src_sizes = src_sizes;
    P.dst_base = dst; P.dst_offsets = dst_off; P.dst_caps = dst_caps;
    P.out_sizes = out_sizes; P.decoded = decoded; P.lz4s = lz4s; P.snappy = snappy;
    std::vector<uint64_t> base(n + 1, 0);
    for (uint32_t i = 0; i < n; i++) base[i + 1] = base[i] + (lz4s ? src_sizes[i] / 2 : src_sizes[i] / 3) + 1;
    std::vector<LzcHead> heads(n);
    memset(heads.data(), 0xCD, sizeof(LzcHead) * (size_t)n);
    std::vector<LzcRec> recs(base[n] + 1);
    memset(recs.data(), 0xCD, sizeof(LzcRec) * recs.size());
    P.c0 = 0; P.nchunks = n; P.heads = heads.data(); P.recs = recs.data(); P.rec_base = base.data();
    emu::launch((n + 31) / 32, 32, 0, [&]() {
        const uint32_t i = blockIdx.x * 32 + threadIdx.x;
        if (i < P.nchunks) lzc_walk_lane(P, i);
    });
    emu::launch((n + 3) / 4, 4 * 32, 0, [&]() {
        const uint32_t i = blockIdx.x * 4 + (threadIdx.x >> 5);
        if (i < P.nchunks) lzc_emit_warp(P, i, threadIdx.x & 31);
    });
    return 0;
}
}
