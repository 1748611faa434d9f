// tests/emu/emu_inflate.cpp -- the inflate kernels (b2c_inflate.cuh: walk, exec, checksum) under the SIMT emulator.
// TEST INFRASTRUCTURE ONLY.
#include "simt_emu.h"

// per-halfword unsigned a >= b: 0xffff where true (the SIMD intrinsic the walk's table lookup uses)
static inline unsigned __vcmpgeu2(unsigned a, unsigned b) {
    return ((a & 0xffffu) >= (b & 0xffffu) ? 0xffffu : 0u) | ((a >> 16) >= (b >> 16) ? 0xffff0000u : 0u);
}

#include "../../compress_b200/csrc/b2c_inflate.cuh"
#include <vector>

using namespace b2c;

extern "C" {

void emu_inflate_set_lane_order(int desc) { emu::lane_order_desc = desc; }

// The device's three kernels over the host call's layout: inputs at src + src_off[i] (src_sizes[i] bytes), contents at
// dst + dst_off[i] (at most dst_caps[i] bytes), records at the bounds b2c_flate_decode_chunks uses.
int emu_inflate(int format, int multistream, const uint8_t *src, const uint64_t *src_off, const uint32_t *src_sizes, uint32_t n,
                uint8_t *dst, const uint64_t *dst_off, const uint32_t *dst_caps, int64_t *out_sizes) {
    InfParams P;
    memset(&P, 0, sizeof(P));
    P.src_base = src; P.src_offsets = src_off; P.src_sizes = src_sizes;
    P.dst_base = dst; P.dst_offsets = dst_off; P.dst_caps = dst_caps;
    P.out_sizes = out_sizes; P.format = format; P.multistream = multistream;
    std::vector<uint64_t> base(n + 1, 0);
    for (uint32_t i = 0; i < n; i++) base[i + 1] = base[i] + inf_rec_cap(src_sizes[i], dst_caps[i]);
    std::vector<InfHead> heads(n);
    memset(heads.data(), 0xCD, sizeof(InfHead) * (size_t)n);
    std::vector<InfRec> recs(base[n] + 1);
    memset(recs.data(), 0xCD, sizeof(InfRec) * recs.size());
    P.c0 = 0; P.nchunks = n; P.heads = heads.data(); P.recs = recs.data(); P.rec_base = base.data();
    const uint32_t nb = (n + INF_WALK_LANES - 1) / INF_WALK_LANES;
    std::vector<InfLane> lanes((size_t)nb * INF_WALK_LANES);        // each CTA's shared memory
    memset(lanes.data(), 0xCD, sizeof(InfLane) * lanes.size());
    InfFixed fixed;
    inf_fixed_build(&fixed, lanes[0].len);
    emu::launch(nb, INF_WALK_LANES, 0, [&]() {
        const uint32_t i = blockIdx.x * INF_WALK_LANES + threadIdx.x;
        if (i < P.nchunks) inf_walk_lane(P, i, &lanes[i], &fixed);
    });
    emu::launch((n + 3) / 4, 4 * 32, 0, [&]() {
        const uint32_t i = blockIdx.x * 4 + (threadIdx.x >> 5);
        if (i < P.nchunks) inf_exec_warp(P, i, threadIdx.x & 31);
    });
    uint32_t tab[256];
    inf_crc_table(tab, 0, 1);
    emu::launch((n + 3) / 4, 4 * 32, 0, [&]() {
        const uint32_t i = blockIdx.x * 4 + (threadIdx.x >> 5);
        if (i < P.nchunks) inf_check_warp(P, i, tab, threadIdx.x & 31);
    });
    return 0;
}
}
