// tests/emu/emu_deflate.cpp -- the stateless deflate kernels (b2c_deflate.cuh: parse, encode, crc) under the SIMT
// emulator, over the launch plan of b2c_flate_stateless_chunks (block slots in passes).  TEST INFRASTRUCTURE ONLY.
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

void emu_deflate_set_lane_order(int desc) { emu::lane_order_desc = desc; }

// The device's kernels over the host call's layout: input i at src + src_off[i] (src_sizes[i] bytes), its dict (dict_sizes
// null: none) at dict + dict_off[i], its output at dst + dst_off[i] (at most dst_caps[i] bytes).  pass_slots: the block
// slots per pass (the library uses 8 192; smaller values make inputs span passes).
int emu_deflate(int format, const uint8_t *src, const uint64_t *src_off, const uint32_t *src_sizes, const uint8_t *eof,
                const uint8_t *dict, const uint64_t *dict_off, const uint32_t *dict_sizes, const uint8_t *hdr, uint32_t hlen,
                uint32_t n, uint8_t *dst, const uint64_t *dst_off, const uint32_t *dst_caps, int64_t *out_sizes,
                uint32_t *crc_out, uint32_t pass_slots) {
    DflParams P;
    memset(&P, 0, sizeof(P));
    P.src_base = src; P.src_offsets = src_off; P.src_sizes = src_sizes; P.eof = eof;
    P.dict_base = dict; P.dict_offsets = dict_off; P.dict_sizes = dict_sizes;
    P.dst_base = dst; P.dst_offsets = dst_off; P.dst_caps = dst_caps;
    P.out_sizes = out_sizes; P.crc_out = crc_out; P.hdr = hdr; P.hlen = hlen; P.format = format;
    uint32_t mb = 1;
    for (uint32_t i = 0; i < n; i++) {
        const uint32_t d = dict_sizes ? (dict_sizes[i] > DFL_DICT ? DFL_DICT : dict_sizes[i]) : 0;
        const uint32_t b = dfl_blocks(src_sizes[i], d);
        if (b > mb) mb = b;
    }
    P.max_blocks = mb;
    const uint64_t total = (uint64_t)n * mb, per = total < pass_slots ? total : pass_slots;
    std::vector<DflState> state(n);
    memset(state.data(), 0xCD, sizeof(DflState) * (size_t)n);
    std::vector<DflSlot> slots(per);
    std::vector<uint32_t> tokens((size_t)per * DFL_SLOT_TOKENS);
    P.state = state.data(); P.slots = slots.data(); P.tokens = tokens.data();
    for (uint32_t i = 0; i < n; i++) out_sizes[i] = 0x7fffffff;
    for (uint64_t g0 = 0; g0 < total; g0 += per) {
        P.g0 = g0; P.g1 = g0 + per < total ? g0 + per : total;
        memset(slots.data(), 0xCD, sizeof(DflSlot) * slots.size());
        const uint32_t i0 = (uint32_t)(P.g0 / mb), i1 = (uint32_t)((P.g1 + mb - 1) / mb);
        const unsigned grid = (unsigned)((P.g1 - P.g0 + 1) / 2);
        std::vector<int16_t> table((size_t)grid * 2 * (1 << 13));         // each CTA's shared memory
        emu::launch(grid, 2 * 32, 0, [&]() {
            const uint64_t g = P.g0 + (uint64_t)blockIdx.x * 2 + (threadIdx.x >> 5);
            if (g < P.g1) dfl_parse_warp(P, g, n, &table[((size_t)blockIdx.x * 2 + (threadIdx.x >> 5)) << 13], threadIdx.x & 31);
        });
        emu::launch((i1 - i0 + 63) / 64, 64, 0, [&]() {
            const uint32_t i = i0 + blockIdx.x * 64 + threadIdx.x;
            if (i < i1) dfl_encode_lane(P, i);
        });
    }
    uint32_t tab[256];
    inf_crc_table(tab, 0, 1);
    emu::launch((n + 3) / 4, 4 * 32, 0, [&]() {
        const uint32_t i = blockIdx.x * 4 + (threadIdx.x >> 5);
        if (i < n) dfl_crc_warp(P, i, tab, threadIdx.x & 31);
    });
    return 0;
}
}
