// tests/emu/emu_flate_best_speed.cpp -- the BestSpeed kernels (b2c_deflate.cuh: l1, l1_check) under the SIMT emulator,
// over the launch plan of b2c_flate_best_speed_chunks (inputs in passes).  TEST INFRASTRUCTURE ONLY.
// Built with -ffp-contract=off: the explicitly rounded intrinsics below are plain IEEE operations.
#include <cstring>
#include "simt_emu.h"

static inline float __fmul_rn(float a, float b) { return a * b; }
static inline float __fadd_rn(float a, float b) { return a + b; }
static inline float __fsub_rn(float a, float b) { return a - b; }
static inline float __fdiv_rn(float a, float b) { return a / b; }
static inline double __dmul_rn(double a, double b) { return a * b; }
static inline double __dadd_rn(double a, double b) { return a + b; }
static inline double __dsub_rn(double a, double b) { return a - b; }
static inline double __ddiv_rn(double a, double b) { return a / b; }
static inline int __float_as_int(float f) { int v; memcpy(&v, &f, 4); return v; }
static inline float __int_as_float(int v) { float f; memcpy(&f, &v, 4); return f; }
static inline unsigned __vcmpgeu2(unsigned a, unsigned b) {
    return ((a & 0xffffu) >= (b & 0xffffu) ? 0xffffu : 0u) | ((a >> 16) >= (b >> 16) ? 0xffff0000u : 0u);
}

#include "../../compress_b200/csrc/b2c_deflate.cuh"
#include <vector>

using namespace b2c;

extern "C" {

void emu_best_speed_set_lane_order(int desc) { emu::lane_order_desc = desc; }

// The BestSpeed kernels' lane and warp functions over the layout of b2c_flate_best_speed_chunks: input i at src +
// src_off[i] (src_sizes[i] bytes), its output at dst + dst_off[i] (at most dst_caps[i] bytes); lanes: the inputs per pass (the library fits as many as 4 GiB
// of scratch holds; smaller values make a batch span passes).  Each pass's tables are zeroed before it, as the library's
// memset does.
int emu_flate_best_speed(int format, const uint8_t *src, const uint64_t *src_off, const uint32_t *src_sizes,
                         const uint8_t *hdr, uint32_t hlen, uint32_t n, uint8_t *dst, const uint64_t *dst_off,
                         const uint32_t *dst_caps, int64_t *out_sizes, uint32_t *check_out, uint32_t lanes) {
    DflParams P;
    memset(&P, 0, sizeof(P));
    P.src_base = src; P.src_offsets = src_off; P.src_sizes = src_sizes;
    P.dst_base = dst; P.dst_offsets = dst_off; P.dst_caps = dst_caps;
    P.out_sizes = out_sizes; P.crc_out = check_out; P.hdr = hdr; P.hlen = hlen; P.format = format;
    std::vector<int32_t> tables((size_t)lanes * DFL_L1_TABLE);
    std::vector<uint32_t> tokens((size_t)lanes * DFL_L1_TOKENS);
    std::vector<DflSlot> slots(lanes);
    std::vector<DflState> state(lanes);
    memset(slots.data(), 0xCD, sizeof(DflSlot) * slots.size());
    memset(state.data(), 0xCD, sizeof(DflState) * state.size());
    P.tokens = tokens.data(); P.slots = slots.data(); P.state = state.data();
    for (uint32_t i = 0; i < n; i++) out_sizes[i] = 0x7fffffff;
    for (uint32_t i0 = 0; i0 < n; i0 += lanes) {
        const uint32_t i1 = n - i0 < lanes ? n : i0 + lanes;
        memset(tables.data(), 0, sizeof(int32_t) * tables.size());
        emu::launch((i1 - i0 + 63) / 64, 64, 0, [&]() {
            const uint32_t i = i0 + blockIdx.x * 64 + threadIdx.x;
            if (i < i1) dfl_l1_lane(P, i, i - i0, tables.data() + (size_t)(i - i0) * DFL_L1_TABLE);
        });
    }
    uint32_t tab[256];
    inf_crc_table(tab, 0, 1);
    emu::launch((n + 3) / 4, 4 * 32, 0, [&]() {
        const uint32_t i = blockIdx.x * 4 + (threadIdx.x >> 5);
        if (i < n) dfl_l1_check_warp(P, i, tab, threadIdx.x & 31);
    });
    return 0;
}
}
