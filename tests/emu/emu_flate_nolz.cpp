// tests/emu/emu_flate_nolz.cpp -- the HuffmanOnly / NoCompression kernels (b2c_deflate.cuh: nolz analyse, plan, emit,
// finish) under the SIMT emulator, over the launch plan of b2c_flate_nolz_chunks (whole inputs per pass).  TEST
// INFRASTRUCTURE ONLY.  Shared memory is the emulator's per-CTA buffer, poisoned before each CTA as the device leaves it
// undefined.  Built with -ffp-contract=off: the explicitly rounded intrinsics below are plain IEEE operations.
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

void emu_nolz_set_lane_order(int desc) { emu::lane_order_desc = desc; }

// The four kernels' device functions over the layout of b2c_flate_nolz_chunks: input i at src + src_off[i]
// (src_sizes[i] bytes), its output at dst + dst_off[i] (at most dst_caps[i] bytes); inputs: the inputs per pass (the
// library fits as many as 4 GiB of records holds; smaller values make a batch span passes).  check_out may be null.
int emu_flate_nolz(int level, int format, const uint8_t *src, const uint64_t *src_off, const uint32_t *src_sizes,
                   const uint8_t *hdr, uint32_t hlen, uint32_t n, uint8_t *dst, const uint64_t *dst_off,
                   const uint32_t *dst_caps, int64_t *out_sizes, uint32_t *check_out, uint32_t inputs) {
    DflNolzParams P;
    memset(&P, 0, sizeof(P));
    P.src_base = src; P.src_offsets = src_off; P.src_sizes = src_sizes;
    P.dst_base = dst; P.dst_offsets = dst_off; P.dst_caps = dst_caps;
    P.out_sizes = out_sizes; P.crc_out = check_out; P.hdr = hdr; P.hlen = hlen; P.format = format; P.level = level;
    uint32_t mw = 1;
    for (uint32_t i = 0; i < n; i++) {
        const uint32_t w = dfl_nolz_windows(src_sizes[i], level);
        if (w > mw) mw = w;
    }
    P.max_windows = mw;
    std::vector<DflNolzWin> wins((size_t)inputs * mw);
    P.wins = wins.data();
    for (uint32_t i = 0; i < n; i++) out_sizes[i] = 0x7fffffff;
    const size_t smemA = sizeof(DflState) + 4 * (256 + 2 * DFL_NOLZ_THREADS / 32 + 256);
    const size_t smemE = 4 * (DFL_NOLZ_STAGE_WORDS + DFL_EOB + 1 + DFL_NOLZ_THREADS / 32);
    for (uint32_t i0 = 0; i0 < n; i0 += inputs) {
        P.i0 = i0; P.i1 = n - i0 < inputs ? n : i0 + inputs;
        const uint64_t slots = (uint64_t)(P.i1 - P.i0) * mw;
        memset(wins.data(), 0xCD, sizeof(DflNolzWin) * wins.size());
        emu::launch((unsigned)slots, DFL_NOLZ_THREADS, smemA, [&]() {
            DflState *st = reinterpret_cast<DflState *>(emu::dyn_smem);
            uint32_t *hist = reinterpret_cast<uint32_t *>(emu::dyn_smem + sizeof(DflState)), *terms = hist + 256,
                     *tab = terms + 2 * DFL_NOLZ_THREADS / 32;
            inf_crc_table(tab, threadIdx.x, blockDim.x);
            dfl_nolz_analyse(P, blockIdx.x, st, hist, terms, tab, threadIdx.x);
        });
        emu::launch((P.i1 - P.i0 + 3) / 4, 4 * 32, 0, [&]() {
            const uint32_t i = P.i0 + blockIdx.x * 4 + (threadIdx.x >> 5);
            if (i < P.i1) dfl_nolz_plan_warp(P, i, threadIdx.x & 31);
        });
        emu::launch((unsigned)slots, DFL_NOLZ_THREADS, smemE, [&]() {
            uint32_t *stage = reinterpret_cast<uint32_t *>(emu::dyn_smem), *codes = stage + DFL_NOLZ_STAGE_WORDS,
                     *wsum = codes + DFL_EOB + 1;
            dfl_nolz_emit(P, blockIdx.x, stage, codes, wsum, threadIdx.x);
        });
        if (level != 0)
            emu::launch((unsigned)((slots + 255) / 256), 256, 0, [&]() {
                const uint64_t g = (uint64_t)blockIdx.x * 256 + threadIdx.x;
                if (g < slots) dfl_nolz_finish(P, g);
            });
    }
    return 0;
}
}
