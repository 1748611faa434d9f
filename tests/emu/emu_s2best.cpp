// tests/emu/emu_s2best.cpp -- the S2 best block encoders (b2c_lz_s2_best_kernel / b2c_lz_snappy_best_kernel, b2c_lz.cuh)
// under the SIMT emulator.  TEST INFRASTRUCTURE ONLY.
#include "simt_emu.h"
#include "../../compress_b200/csrc/b2c_lz.cuh"
#include <vector>

using namespace b2c;

extern "C" {

void emu_s2best_set_lane_order(int desc) { emu::lane_order_desc = desc; }

// S2 (snappy = 0) / Snappy-compatible (snappy = 1) best encode of nchunks chunks (chunk i = src + i * stride, sizes[i]
// bytes) into slots of dst_stride bytes; out_sizes[i] = bytes written or a negative error, as on the device
int emu_s2best_encode(const uint8_t *src, uint64_t stride, const uint32_t *sizes, uint32_t nchunks, uint8_t *dst,
                      uint64_t dst_stride, int64_t *out_sizes, int snappy) {
    std::vector<uint8_t> scratch(LzLayout<LZ_S2BEST>::SCRATCH_BYTES, 0xCD);
    ZstdEncParams P;
    memset(&P, 0, sizeof(P));
    P.src_base = src; P.src_stride = stride; P.src_sizes = sizes;
    P.dst_base = dst; P.dst_stride = dst_stride; P.dst_cap = (uint32_t)dst_stride;
    P.out_sizes = out_sizes; P.nchunks = nchunks; P.scratch = scratch.data(); P.blockmax = 65536;
    emu::launch(1, LzCfg<LZ_S2BEST>::NT, LzLayout<LZ_S2BEST>::SMEM_BYTES, [&]() {
        for (uint32_t c = 0; c < P.nchunks; c++) {
            if (snappy) lz_parse_chunk<LZ_S2BEST, LZ_MODE_SNAPPY>(emu::dyn_smem, P, c, P.scratch);
            else lz_parse_chunk<LZ_S2BEST, LZ_MODE_S2>(emu::dyn_smem, P, c, P.scratch);
        }
    });
    return 0;
}
}
