// compress_b200/csrc/b2c_api.cu -- C ABI (include/b2c.h) over the sm_90a kernels.
// Plain CUDA runtime: no torch types cross this boundary.  No CPU fallback: without a device
// every call fails with B2C_ERR_NO_DEVICE.
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
#include <thread>
#include <mutex>
#include <condition_variable>
#include <deque>
#include <chrono>
#include <atomic>
#include "../../include/b2c.h"
#include "b2c_zstd_enc.cuh"
#include "b2c_lz.cuh"
#include "b2c_frame.cuh"
#include "b2c_zstd_dec.cuh"
#include "b2c_zstd_dec_staged.cuh"
#include "b2c_s2_dec.cuh"
#include "b2c_s2_stream.cuh"
#include "b2c_huf0.cuh"
#include "b2c_lz4_cvt.cuh"
#include "b2c_inflate.cuh"
#include "b2c_deflate.cuh"

#ifndef TABLES_CTAS_PER_SM
#define TABLES_CTAS_PER_SM TABLES_MIN_CTAS   // K2: resident CTAs per SM (44 KB static shared memory each)
#endif

using namespace b2c;

// Memory the context owns: device or pinned host memory, grown by reserve() and freed with the context.  Every member
// states where it lives and how it grows where it is declared.  cap is in bytes.
enum BufKind { kDevice, kPinned };
enum BufGrowth { kExact, kHeadroom };   // kHeadroom: 25 % more than asked for, so that slowly rising sizes do not regrow each call
template <class T = uint8_t> struct Buf {
    const BufKind kind;
    const BufGrowth growth;
    T *p = nullptr;
    size_t cap = 0;
    Buf(BufKind k, BufGrowth g) : kind(k), growth(g) {}
    Buf(const Buf &) = delete;
    Buf &operator=(const Buf &) = delete;
    ~Buf() { if (p) { if (kind == kPinned) cudaFreeHost(p); else cudaFree(p); } }
    template <class U> U *at(size_t off) const { return reinterpret_cast<U *>(reinterpret_cast<uint8_t *>(p) + off); }
};
// An event or stream the context owns, destroyed with it.
template <class H, cudaError_t (*destroy)(H)> struct Owned {
    H h = nullptr;
    Owned() = default;
    Owned(const Owned &) = delete;
    Owned &operator=(const Owned &) = delete;
    ~Owned() { if (h) destroy(h); }
    operator H() const { return h; }
};
using Event = Owned<cudaEvent_t, cudaEventDestroy>;
using Stream = Owned<cudaStream_t, cudaStreamDestroy>;

// One slot of the encode pipeline.  b2c_zstd_encode_packed alternates batches between the two slots (H2D / kernels / D2H
// overlap); every other encode call uses slot 0.  The host-buffer buffers hold max_chunks chunks of 64 KiB.
struct EncSlot {
    Buf<> d_in{kDevice, kExact}, d_out{kDevice, kExact};      // input chunks | output slots of kSlot bytes
    Buf<> d_packed{kDevice, kExact};                          // the batch's frames back to back
    Buf<int64_t> d_sizes{kDevice, kExact}, h_sizes{kPinned, kExact};   // h_sizes: sizes | packed offsets
    Buf<uint64_t> d_offsets{kDevice, kExact};
    Buf<uint32_t> d_src_sizes{kDevice, kExact}, h_src_sizes{kPinned, kExact};
    Buf<> h_in{kPinned, kExact}, h_out{kPinned, kExact};      // pinned staging (slot 1's: allocated for the first pageable caller)
    Buf<ChunkWork> work{kDevice, kExact};                     // per-chunk work records, grown on demand
    Buf<> pool{kDevice, kExact};                              // per-chunk work pool slabs (literals, sequences, codes, state bits)
    size_t scratch_off = 0;                                   // this slot's set of the per-CTA parse scratch
    Event ev, ev_in, ev_out;                                  // compute / H2D / D2H of the slot's batch finished
};

struct b2c_ctx {
    int device = 0;
    int sm_count = 0;
    size_t max_chunks = 0;
    Stream stream;                      // every host-buffer call; the kernels of b2c_zstd_encode_packed
    Stream stream2, stream3;            // b2c_zstd_encode_packed: H2D / D2H
    Stream dec_aux;                     // staged decode: the literal kernel runs beside the sequence walk
    Event ev_busy;                      // last launch that used the context's scratch / work buffers
    cudaStream_t busy_stream = nullptr; bool busy_valid = false;
    Event dec_fork, dec_join;
    Buf<> d_scratch{kDevice, kExact};   // per-CTA parse scratch (two sets: one per pipeline slot)
    EncSlot slot[2];
    Buf<> d_fr{kDevice, kExact};        // frame mode: block / frame tables, block slots (grown on demand)
    Buf<> d_fr_io{kDevice, kExact};     // frame mode, host-buffer call: staged input | packed output | results
    Buf<> d_s2d{kDevice, kHeadroom};    // staged S2 block decode: block heads + element records
    Buf<> d_lzc{kDevice, kHeadroom};    // LZ4 -> S2 conversion: block heads + sequence records of one pass
    Buf<> d_inf{kDevice, kHeadroom};    // inflate: input heads + match / stored-run / member records of one pass
    Buf<> d_dfl{kDevice, kHeadroom};    // stateless deflate: per-input writer state | gzip header | block slots of one pass
    Buf<> d_s2best{kDevice, kExact};    // S2 best parse scratch (four candidates per position), reserved on first use
    Buf<> d_s2s{kDevice, kExact};       // S2 stream calls: block slots, sizes, checksums, scan, tables (grown on demand)
    Buf<> d_s2s_io{kDevice, kExact};    //   host-buffer calls: staged input | output
    Buf<uint32_t> d_counters{kDevice, kExact}; uint32_t counter_seq = 0;   // chunk counters of the persistent parse kernels (one per launch, rotating)
    int enc_fused_xxh = 1;                                 // B2C_ENC_XXH=kernel: XXH64 as its own kernel (A/B measurements)
    // decoder: per-warp literal scratch, host-path staging (grown on demand)
    Buf<> d_dec_lit{kDevice, kHeadroom};
    Buf<> d_fd{kDevice, kHeadroom};                        // staged decoder: records | FSE tables | Huffman tables
    Buf<uint32_t> d_fd_const{kDevice, kExact};             //   code maps + predefined tables
    Buf<> d_fd_seq{kDevice, kHeadroom};                    //   sequence records
    Buf<> d_fd_lit{kDevice, kHeadroom};                    //   decoded literals
    int dec_staged = 1;                                    // B2C_DEC=onewarp: one-warp decoder only (A/B measurements)
    bool fd_last = false, s2d_last = false;                // d_fd / d_s2d hold the records of the most recent zstd / S2 decode launch
    float dec_ms[6] = {0, 0, 0, 0, 0, 0}; Event dec_ev[7]; int dec_prof = 0;
    Buf<> d_dec_in{kDevice, kHeadroom}, d_dec_out{kDevice, kHeadroom}, d_dec_meta{kDevice, kHeadroom};
    Buf<> h_stg_in{kPinned, kHeadroom}, h_stg_out{kPinned, kHeadroom};   // pinned staging of the pointer-table calls
    // optional per-kernel timing of the encode pipeline (b2c_profile_*): 6 events per encode call
    bool prof = false;
    std::vector<cudaEvent_t> pev;
    size_t pev_used = 0;
    uint64_t launches = 0;
    char err[256] = {0};
    ~b2c_ctx() { for (cudaEvent_t e : pev) cudaEventDestroy(e); }
};

#define CK(call)                                                                                       \
    do {                                                                                               \
        cudaError_t e_ = (call);                                                                       \
        if (e_ != cudaSuccess) {                                                                       \
            if (ctx) snprintf(ctx->err, sizeof(ctx->err), "%s: %s", #call, cudaGetErrorString(e_));    \
            return B2C_ERR_CUDA;                                                                       \
        }                                                                                              \
    } while (0)

// Grows b to at least `need` bytes; its contents are not kept.  A device buffer is replaced only after the device has
// synchronised: kernels of earlier calls on other streams may still use the old one.
template <class T> static int reserve(b2c_ctx *ctx, Buf<T> &b, size_t need) {
    if (b.cap >= need) return B2C_OK;
    const bool dev = b.kind == kDevice;
    if (dev) CK(cudaDeviceSynchronize());
    if (b.p) CK(dev ? cudaFree(b.p) : cudaFreeHost(b.p));
    b.p = nullptr; b.cap = 0;
    if (b.growth == kHeadroom) need += need / 4;
    CK(dev ? cudaMalloc(&b.p, need) : cudaMallocHost(&b.p, need));
    b.cap = need;
    return B2C_OK;
}

// Pieces of one buffer, each starting 256-byte aligned: take() returns a piece's offset, end is the bytes they span.
struct Layout {
    size_t end = 0;
    size_t take(size_t bytes) { const size_t r = end; end += (bytes + 255) & ~(size_t)255; return r; }
};

// Host-side gather / scatter of many separately addressed pieces (the pointer-table calls): index ranges are spread over a few
// host threads when there is enough to move -- one thread copies about 10 GB/s, which otherwise bounds these calls far
// below the PCIe rate.  fn(i) handles piece i; pieces are independent.
template <class F> static void parallel_pieces(size_t n, size_t total_bytes, F fn) {
    unsigned hw = std::thread::hardware_concurrency();
    unsigned nt = hw ? (hw < 8 ? hw : 8) : 4;
    if (total_bytes < ((size_t)8 << 20) || n < 2 * (size_t)nt || nt < 2) { for (size_t i = 0; i < n; i++) fn(i); return; }
    const size_t per = (n + nt - 1) / nt;
    std::vector<std::thread> th;
    for (unsigned t = 1; t < nt; t++) {
        const size_t lo = (size_t)t * per, hi = lo + per < n ? lo + per : n;
        if (lo >= n) break;
        th.emplace_back([=]() { for (size_t i = lo; i < hi; i++) fn(i); });
    }
    for (size_t i = 0; i < (per < n ? per : n); i++) fn(i);
    for (auto &x : th) x.join();
}

static const uint32_t kSlot = 65536 + 512;  // >= MaxEncodedSize(65536) = 65536 + 3 + 7 + 4, 16-byte multiple

// ---- small helper kernels -------------------------------------------------------------------
// exclusive scan of the (non-negative) chunk sizes -> packed offsets; single CTA
__global__ void b2c_scan_sizes_kernel(const int64_t *sizes, uint64_t *offsets, uint32_t n) {
    __shared__ uint64_t carry;
    __shared__ uint64_t wsum[32];
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (uint32_t base = 0; base < n; base += blockDim.x) {
        uint32_t i = base + threadIdx.x;
        uint64_t v = (i < n && sizes[i] > 0) ? (uint64_t)sizes[i] : 0;
        uint64_t incl = v;
        for (int d = 1; d < 32; d <<= 1) {
            uint64_t t = __shfl_up_sync(0xffffffffu, incl, d);
            if ((threadIdx.x & 31) >= (unsigned)d) incl += t;
        }
        if ((threadIdx.x & 31) == 31) wsum[threadIdx.x >> 5] = incl;
        __syncthreads();
        if (threadIdx.x < 32) {
            uint64_t x = (threadIdx.x < (blockDim.x >> 5)) ? wsum[threadIdx.x] : 0, xi = x;
            for (int d = 1; d < 32; d <<= 1) {
                uint64_t t = __shfl_up_sync(0xffffffffu, xi, d);
                if (threadIdx.x >= (unsigned)d) xi += t;
            }
            wsum[threadIdx.x] = xi - x;
        }
        __syncthreads();
        uint64_t ex = carry + wsum[threadIdx.x >> 5] + incl - v;
        if (i < n) offsets[i] = ex;
        __syncthreads();
        if (threadIdx.x == blockDim.x - 1) carry = ex + v;
        __syncthreads();
    }
    if (threadIdx.x == 0) offsets[n] = carry;
}
// copy chunk i's bytes from its slot to packed[offsets[i]]
__global__ void b2c_pack_kernel(const uint8_t *slots, uint64_t slot_stride, const int64_t *sizes,
                                const uint64_t *offsets, uint8_t *packed, uint32_t n) {
    for (uint32_t c = blockIdx.x; c < n; c += gridDim.x) {
        int64_t sz = sizes[c];
        if (sz <= 0) continue;
        const uint8_t *s = slots + (uint64_t)c * slot_stride;
        uint8_t *d = packed + offsets[c];
        uint32_t head = (uint32_t)((16 - (reinterpret_cast<uintptr_t>(d) & 15)) & 15);
        if (head > (uint32_t)sz) head = (uint32_t)sz;
        for (uint32_t i = threadIdx.x; i < head; i += blockDim.x) d[i] = s[i];
        // aligned body: 4-byte stores assembled from (possibly unaligned) source words
        uint32_t body = ((uint32_t)sz - head) & ~3u;
        for (uint32_t i = threadIdx.x * 4; i < body; i += blockDim.x * 4) {
            uint32_t v = ld32u(s, head + i);
            *reinterpret_cast<uint32_t *>(d + head + i) = v;
        }
        for (uint32_t i = head + body + threadIdx.x; i < (uint32_t)sz; i += blockDim.x) d[i] = s[i];
    }
}

// ---- context -----------------------------------------------------------------------------------
extern "C" {

int b2c_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
    return n;
}

b2c_ctx *b2c_ctx_create(int device, size_t max_chunks) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0 || device >= n) return nullptr;
    if (cudaSetDevice(device) != cudaSuccess) return nullptr;
    b2c_ctx *ctx = new b2c_ctx();
    ctx->device = device;
    ctx->max_chunks = max_chunks;
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) { delete ctx; return nullptr; }
    ctx->sm_count = prop.multiProcessorCount;
    bool ok = true;
    size_t scratch_slot = 0;            // bytes of one slot's scratch set
    {
        size_t a = 0;
        size_t b = (size_t)ctx->sm_count * LzCfg<1>::MIN_CTAS * LzLayout<1>::SCRATCH_BYTES;
        size_t c = (size_t)ctx->sm_count * LzCfg<2>::MIN_CTAS * LzLayout<2>::SCRATCH_BYTES;
        size_t d3 = (size_t)ctx->sm_count * LzCfg<3>::MIN_CTAS * LzLayout<3>::SCRATCH_BYTES;
        size_t d4 = (size_t)ctx->sm_count * LzCfg<4>::MIN_CTAS * LzLayout<4>::SCRATCH_BYTES;
        if (d3 > a) a = d3;
        if (d4 > a) a = d4;
        size_t d5 = (size_t)ctx->sm_count * LzCfg<5>::MIN_CTAS * LzLayout<5>::SCRATCH_BYTES;
        if (d5 > a) a = d5;
        scratch_slot = ((a > b ? (a > c ? a : c) : (b > c ? b : c)) + 255) & ~(size_t)255;
    }
    ok = ok && reserve(ctx, ctx->d_scratch, 2 * scratch_slot) == B2C_OK;
    ok = ok && cudaEventCreateWithFlags(&ctx->ev_busy.h, cudaEventDisableTiming) == cudaSuccess;
    const struct { const void *fn; int bytes; } smem[] = {
        {(const void *)b2c_lz_parse1_kernel, (int)LzLayout<1>::SMEM_BYTES},
        {(const void *)b2c_lz_parse2_kernel, (int)LzLayout<2>::SMEM_BYTES},
        {(const void *)b2c_lz_parse3_kernel, (int)LzLayout<5>::SMEM_BYTES},
        {(const void *)b2c_lz_s2_fast_kernel, (int)LzLayout<3>::SMEM_BYTES},
        {(const void *)b2c_lz_snappy_fast_kernel, (int)LzLayout<3>::SMEM_BYTES},
        {(const void *)b2c_lz_s2_better_kernel, (int)LzLayout<4>::SMEM_BYTES},
        {(const void *)b2c_lz_snappy_better_kernel, (int)LzLayout<4>::SMEM_BYTES},
        {(const void *)b2c_lz_s2_best_kernel, (int)LzLayout<LZ_S2BEST>::SMEM_BYTES},
        {(const void *)b2c_lz_snappy_best_kernel, (int)LzLayout<LZ_S2BEST>::SMEM_BYTES},
        {(const void *)b2c_zstd_hist_kernel, (int)HIST_SMEM_BYTES},
        {(const void *)b2c_zstd_pack128_kernel, (int)PackCfg<131072>::SMEM_BYTES},
        {(const void *)b2c_zstd_pack_kernel, (int)PACK_SMEM_BYTES},
        {(const void *)b2c_zstd_chains_kernel, (int)CHAIN_SMEM_BYTES},
        {(const void *)b2c_huf_compress_kernel, (int)HUF0_SMEM_BYTES},
        {(const void *)b2c_huf_decompress_kernel, (int)DEC_SMEM_BYTES},
        {(const void *)b2c_huf_dec_prep_kernel, (int)DEC_SMEM_BYTES},
        {(const void *)b2c_huf_read_table_kernel, (int)DEC_SMEM_BYTES},
        {(const void *)b2c_zstd_decode_kernel, (int)DEC_SMEM_BYTES},
        {(const void *)b2c_zstd_dec_lit_kernel, (int)(FD_LIT_WARPS * FD_LIT_WARP_BYTES)},
        {(const void *)b2c_zstd_dec_init_kernel, (int)DEC_WARP_BYTES},
    };
    for (const auto &k : smem)
        ok = ok && cudaFuncSetAttribute(k.fn, cudaFuncAttributeMaxDynamicSharedMemorySize, k.bytes) == cudaSuccess;
    // at most two chains CTAs per SM, the rest of the SM's memory stays L1: a 16384-chunk pass (512 CTAs) took
    // 1.21 ms per GiB with four CTAs sharing an SM and 0.99 ms with two (H100 SXM at 700 W, level 1)
    ok = ok && cudaFuncSetAttribute(b2c_zstd_chains_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, 50) == cudaSuccess;
    ok = ok && cudaStreamCreateWithFlags(&ctx->stream.h, cudaStreamNonBlocking) == cudaSuccess;
    ok = ok && reserve(ctx, ctx->d_fd_const, FD_CONST_ENTRIES * sizeof(uint32_t)) == B2C_OK;
    if (ok) {
        b2c_zstd_dec_init_kernel<<<1, 32, DEC_WARP_BYTES>>>(ctx->d_fd_const.p);
        ok = cudaDeviceSynchronize() == cudaSuccess;
    }
    for (Event &e : ctx->dec_ev) ok = ok && cudaEventCreate(&e.h) == cudaSuccess;
    ok = ok && cudaStreamCreateWithFlags(&ctx->dec_aux.h, cudaStreamNonBlocking) == cudaSuccess;
    ok = ok && cudaEventCreateWithFlags(&ctx->dec_fork.h, cudaEventDisableTiming) == cudaSuccess;
    ok = ok && cudaEventCreateWithFlags(&ctx->dec_join.h, cudaEventDisableTiming) == cudaSuccess;
    ok = ok && reserve(ctx, ctx->d_counters, 256 * sizeof(uint32_t)) == B2C_OK;
    {
        const char *es = getenv("B2C_ENC_XXH");
        ctx->enc_fused_xxh = (es && strcmp(es, "kernel") == 0) ? 0 : 1;
    }
    {
        const char *de = getenv("B2C_DEC");
        ctx->dec_staged = (de && strcmp(de, "onewarp") == 0) ? 0 : 1;
    }
    if (ok && max_chunks) {
        ok = ok && cudaStreamCreateWithFlags(&ctx->stream2.h, cudaStreamNonBlocking) == cudaSuccess;
        ok = ok && cudaStreamCreateWithFlags(&ctx->stream3.h, cudaStreamNonBlocking) == cudaSuccess;
    }
    for (int k = 0; k < 2; k++) {
        EncSlot &S = ctx->slot[k];
        S.scratch_off = k * scratch_slot;
        if (!ok || !max_chunks) continue;
        ok = ok && reserve(ctx, S.d_in, max_chunks * (size_t)ENC_MAX_CHUNK) == B2C_OK;
        ok = ok && reserve(ctx, S.d_out, max_chunks * (size_t)kSlot) == B2C_OK;
        ok = ok && reserve(ctx, S.d_packed, max_chunks * (size_t)kSlot) == B2C_OK;
        ok = ok && reserve(ctx, S.d_sizes, max_chunks * sizeof(int64_t)) == B2C_OK;
        ok = ok && reserve(ctx, S.h_sizes, (max_chunks + 1) * sizeof(int64_t) * 2) == B2C_OK;
        ok = ok && reserve(ctx, S.d_offsets, (max_chunks + 1) * sizeof(uint64_t)) == B2C_OK;
        ok = ok && reserve(ctx, S.d_src_sizes, max_chunks * sizeof(uint32_t)) == B2C_OK;
        ok = ok && reserve(ctx, S.h_src_sizes, max_chunks * sizeof(uint32_t)) == B2C_OK;
        if (k == 0) {       // slot 1's staging is allocated by the first pageable caller of b2c_zstd_encode_packed
            ok = ok && reserve(ctx, S.h_in, max_chunks * (size_t)ENC_MAX_CHUNK) == B2C_OK;
            ok = ok && reserve(ctx, S.h_out, max_chunks * (size_t)kSlot) == B2C_OK;
        }
        for (Event *e : {&S.ev, &S.ev_in, &S.ev_out})
            ok = ok && cudaEventCreateWithFlags(&e->h, cudaEventDisableTiming) == cudaSuccess;
    }
    if (!ok) { b2c_ctx_destroy(ctx); return nullptr; }
    return ctx;
}

void b2c_ctx_destroy(b2c_ctx *ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    delete ctx;             // the members free the buffers and destroy the events and streams they hold
}

const char *b2c_strerror(int code) {
    switch (code) {
    case B2C_OK: return "ok";
    case B2C_ERR_NO_DEVICE: return "no CUDA device (libb200comp has no CPU fallback)";
    case B2C_ERR_CUDA: return "CUDA runtime error";
    case B2C_ERR_ARG: return "invalid argument";
    case B2C_ERR_TOO_BIG: return "chunk too big for this level's block size";
    case B2C_ERR_DST_SMALL: return "destination too small";
    case B2C_ERR_CORRUPT: return "corrupt input";
    case B2C_ERR_MAGIC: return "invalid input: magic number mismatch";
    case B2C_ERR_WINDOW: return "window size exceeded";
    case B2C_ERR_CRC: return "CRC check failed";
    case B2C_ERR_SIZE: return "frame size exceeded / mismatch";
    case B2C_ERR_UNSUPPORTED: return "unsupported";
    case B2C_ERR_UNEXPECTED_EOF: return "unexpected end of input";
    default: return "unknown error";
    }
}
const char *b2c_last_cuda_error(b2c_ctx *ctx) { return ctx ? ctx->err : "no context"; }
int b2c_sm_count(b2c_ctx *ctx) { return ctx ? ctx->sm_count : 0; }
uint64_t b2c_launch_count(b2c_ctx *ctx) { return ctx ? ctx->launches : 0; }

int b2c_profile_enable(b2c_ctx *ctx, int on) {
    if (!ctx) return B2C_ERR_NO_DEVICE;
    ctx->prof = on != 0;
    ctx->pev_used = 0;
    return B2C_OK;
}
// ms[k] = summed duration of kernel k (0 xxh64, 1 parse, 2 histograms, 3 tables, 4 chains, 5 pack) over the encode launches issued
// since b2c_profile_enable(ctx, 1); *ncalls = number of encode calls.  Synchronises the device.
int b2c_profile_read(b2c_ctx *ctx, double *ms, uint32_t *ncalls) {
    if (!ctx) return B2C_ERR_NO_DEVICE;
    CK(cudaSetDevice(ctx->device));
    CK(cudaDeviceSynchronize());
    for (int k = 0; k < 6; k++) ms[k] = 0.0;
    for (size_t c = 0; c + 7 <= ctx->pev_used; c += 7)
        for (int k = 0; k < 6; k++) {
            float t = 0.f;
            CK(cudaEventElapsedTime(&t, ctx->pev[c + k], ctx->pev[c + k + 1]));
            ms[k] += (double)t;
        }
    if (ncalls) *ncalls = (uint32_t)(ctx->pev_used / 7);
    ctx->pev_used = 0;
    return B2C_OK;
}

// Decode-side counterpart: ms[0..5] = summed durations of {scan, literals, sequences, execute, xxh64, one-warp decoder} over the
// staged decode launches since b2c_decode_profile_enable(ctx, 1).  Enabled, every decode launch synchronises.
int b2c_decode_profile_enable(b2c_ctx *ctx, int on) {
    if (!ctx) return B2C_ERR_NO_DEVICE;
    ctx->dec_prof = on != 0;
    for (int i = 0; i < 6; i++) ctx->dec_ms[i] = 0.f;
    return B2C_OK;
}
// flags[i] = 1 where the per-input record (whose first word is its state; 0 = finished by the staged kernels) says so.
// last: the most recent launch ran the staged kernels (otherwise the records are an earlier launch's and every flag is 0).
static int staged_flags(b2c_ctx *ctx, const uint8_t *recs, bool last, size_t rec_bytes, size_t cap, uint32_t nchunks, uint8_t *flags) {
    memset(flags, 0, nchunks);
    if (!recs || !last || nchunks == 0) return B2C_OK;
    CK(cudaSetDevice(ctx->device));
    CK(cudaDeviceSynchronize());
    if ((size_t)nchunks * rec_bytes > cap) return B2C_ERR_ARG;
    std::vector<uint32_t> st(nchunks);
    CK(cudaMemcpy2D(st.data(), sizeof(uint32_t), recs, rec_bytes, sizeof(uint32_t), nchunks, cudaMemcpyDeviceToHost));
    for (uint32_t i = 0; i < nchunks; i++) flags[i] = st[i] == 0;
    return B2C_OK;
}
// Per input of the first nchunks of the most recent decode launch: 1 if the staged kernels completed it, 0 if it went
// through the one-warp decoder.  Synchronises the device.  Test / diagnostics hook.
int b2c_decode_staged_flags(b2c_ctx *ctx, uint32_t nchunks, uint8_t *flags) {
    if (!ctx || (!flags && nchunks)) return B2C_ERR_ARG;
    return staged_flags(ctx, ctx->d_fd.p, ctx->fd_last, sizeof(FdChunk), ctx->d_fd.cap, nchunks, flags);
}
// The same for the most recent S2 block decode launch: blocks finished by the staged kernels (tag walk + execution).
int b2c_s2_decode_staged_flags(b2c_ctx *ctx, uint32_t nchunks, uint8_t *flags) {
    if (!ctx || (!flags && nchunks)) return B2C_ERR_ARG;
    return staged_flags(ctx, ctx->d_s2d.p, ctx->s2d_last, sizeof(S2Head), ctx->d_s2d.cap, nchunks, flags);
}
// How many of the first nchunks inputs of the most recent (S2) decode launch the staged kernels completed.
static int staged_count(int (*flags_of)(b2c_ctx *, uint32_t, uint8_t *), b2c_ctx *ctx, uint32_t nchunks, uint32_t *staged) {
    if (!ctx || !staged) return B2C_ERR_ARG;
    std::vector<uint8_t> f(nchunks);
    const int rc = flags_of(ctx, nchunks, f.data());
    *staged = 0;
    for (uint8_t v : f) *staged += v;
    return rc;
}
int b2c_decode_staged_count(b2c_ctx *ctx, uint32_t nchunks, uint32_t *staged) {
    return staged_count(b2c_decode_staged_flags, ctx, nchunks, staged);
}
int b2c_s2_decode_staged_count(b2c_ctx *ctx, uint32_t nchunks, uint32_t *staged) {
    return staged_count(b2c_s2_decode_staged_flags, ctx, nchunks, staged);
}
int b2c_decode_profile_read(b2c_ctx *ctx, double *ms) {
    if (!ctx) return B2C_ERR_NO_DEVICE;
    for (int i = 0; i < 6; i++) { ms[i] = (double)ctx->dec_ms[i]; ctx->dec_ms[i] = 0.f; }
    return B2C_OK;
}

size_t b2c_zstd_bound(size_t size, int level) {
    // Encoder.MaxEncodedSize, zstd/encoder.go:843-873 (crc on)
    size_t blockSize = (level == B2C_LEVEL_FASTEST) ? (1u << 16) : (128u << 10);
    size_t fh = 4 + 2;
    if (size < 256) fh++;
    else if (size < 65536 + 256) fh += 2;
    else if (size < 0x7fffffff) fh += 4;
    else fh += 8;
    fh += 4;
    size_t blocks = (size + blockSize) / blockSize;
    return fh + 3 * blocks + size;
}

// a zeroed chunk counter for one launch of a persistent parse kernel (rotating: launches in flight never share one)
static int next_counter(b2c_ctx *ctx, cudaStream_t st, uint32_t **out) {
    uint32_t *c = ctx->d_counters.p + (ctx->counter_seq++ & 255u);
    CK(cudaMemsetAsync(c, 0, sizeof(uint32_t), st));
    *out = c;
    return B2C_OK;
}

static uint32_t level_block(int level) { return level == B2C_LEVEL_FASTEST ? (1u << 16) : (128u << 10); }
static bool level_ok(int level) { return level == B2C_LEVEL_FASTEST || level == B2C_LEVEL_DEFAULT || level == B2C_LEVEL_BETTER; }
static size_t level_slot(int level) { return (size_t)level_block(level) + 512; }   // >= MaxEncodedSize(block), 16-byte multiple

// Calls that use the context's scratch / work buffers are ordered among themselves even when they are issued on
// different streams: the next one waits for the event the previous one recorded.
static int ctx_order_begin(b2c_ctx *ctx, cudaStream_t st) {
    if (ctx->busy_valid && ctx->busy_stream != st) CK(cudaStreamWaitEvent(st, ctx->ev_busy, 0));
    return B2C_OK;
}
static int ctx_order_end(b2c_ctx *ctx, cudaStream_t st) {
    CK(cudaEventRecord(ctx->ev_busy, st));
    ctx->busy_stream = st; ctx->busy_valid = true;
    return B2C_OK;
}

// One encode launch = the six kernels over at most `sub` chunks at a time (the work records and the work pool are
// sized for `sub` chunks, so a device-resident call of any size needs a bounded amount of scratch).
static int launch_encode(b2c_ctx *ctx, int level, int flags, const void *d_src, size_t src_stride,
                         const uint32_t *d_sizes, uint32_t size_all, void *d_dst, size_t dst_stride,
                         int64_t *d_out_sizes, uint32_t nchunks, uint32_t *dbg_hdr, uint32_t *dbg_seqs,
                         uint8_t *dbg_lits, uint32_t dbg_cap, cudaStream_t st, unsigned long long *dbg_cycles = nullptr,
                         int slot = 0, const EncBlockDesc *d_desc = nullptr) {
    if (!ctx) return B2C_ERR_NO_DEVICE;
    if (!level_ok(level)) return B2C_ERR_UNSUPPORTED;
    if (nchunks == 0) return B2C_OK;
    if (dst_stride > 0xffffffffull) return B2C_ERR_ARG;
    CK(cudaSetDevice(ctx->device));
    const uint32_t blockmax = level_block(level);
    const uint64_t pstride = wk_pool_stride(blockmax);
    // One pass takes a 1 GiB batch (16384 x 64 KiB or 8192 x 128 KiB) in one go: every kernel's drain and tail is paid
    // once, and the persistent parse and the chains kernel have enough chunks to fill the device.  Work pool: 345 KB per
    // 64 KiB chunk (5.7 GB at 16384), 821 KB per 128 KiB block (6.7 GB at 8192); it grows only for calls that large.
    const uint32_t subMax = blockmax > 65536 ? 8192u : 16384u;
    const uint32_t sub = nchunks < subMax ? nchunks : subMax;
    EncSlot &S = ctx->slot[slot];
    { int r = reserve(ctx, S.work, (size_t)sub * sizeof(ChunkWork)); if (r) return r; }
    { int r = reserve(ctx, S.pool, (size_t)sub * pstride); if (r) return r; }
    { int r = ctx_order_begin(ctx, st); if (r) return r; }
    const unsigned sms = (unsigned)ctx->sm_count;
    for (uint32_t c0 = 0; c0 < nchunks; c0 += sub) {
        const uint32_t m = (nchunks - c0 < sub) ? nchunks - c0 : sub;
        ZstdEncParams P;
        memset(&P, 0, sizeof(P));
        P.src_base = d_desc ? (const uint8_t *)d_src : (const uint8_t *)d_src + (size_t)c0 * src_stride; P.src_stride = src_stride;
        P.desc = d_desc ? d_desc + c0 : nullptr;
        P.src_sizes = d_sizes ? d_sizes + c0 : nullptr; P.src_size_all = size_all;
        P.dst_base = (uint8_t *)d_dst + (size_t)c0 * dst_stride; P.dst_stride = dst_stride; P.dst_cap = (uint32_t)dst_stride;
        P.out_sizes = d_out_sizes + c0; P.nchunks = m; P.flags = (uint32_t)flags;
        P.scratch = ctx->d_scratch.p + S.scratch_off;
        P.work = S.work.p;
        P.pool = S.pool.p; P.pool_stride = pstride; P.maxseq = wk_maxseq(blockmax); P.blockmax = blockmax;
        P.big = blockmax > 65536 ? 1u : 0u; P.level = (uint32_t)level;
        if (dbg_hdr) {
            P.dbg_hdr = dbg_hdr + (size_t)c0 * 4; P.dbg_seqs = dbg_seqs + (size_t)c0 * dbg_cap * 3;
            P.dbg_lits = dbg_lits + (size_t)c0 * blockmax; P.dbg_seq_cap = dbg_cap;
        }
        P.dbg_cycles = dbg_cycles ? dbg_cycles + (size_t)c0 * 16 * 32 : nullptr;
        cudaEvent_t *pe = nullptr;
        if (ctx->prof) {
            while (ctx->pev.size() < ctx->pev_used + 7) {
                cudaEvent_t e;
                CK(cudaEventCreate(&e));
                ctx->pev.push_back(e);
            }
            pe = ctx->pev.data() + ctx->pev_used;
            ctx->pev_used += 7;
        }
#define PEV(k) do { if (pe) cudaEventRecord(pe[k], st); } while (0)
        PEV(0);
        // XXH64 rides in the chains launch (four more warps per CTA); as its own kernel only for A/B measurements
        const bool wantXxh = (flags & B2C_ZSTD_FRAME) && (flags & B2C_ZSTD_CRC);
        if (wantXxh && !ctx->enc_fused_xxh) {
            b2c_zstd_xxh_kernel<<<(4 * m + 127) / 128, 128, 0, st>>>(P);
            ctx->launches += 1;
        }
        { int r = next_counter(ctx, st, &P.counter); if (r) return r; }
        PEV(1);
        {
            if (level == B2C_LEVEL_FASTEST) {
                const unsigned cap = sms * LzCfg<1>::MIN_CTAS, g1 = cap < m ? cap : m;
                b2c_lz_parse1_kernel<<<g1, LzCfg<1>::NT, LzLayout<1>::SMEM_BYTES, st>>>(P);
            } else if (level == B2C_LEVEL_DEFAULT) {
                const unsigned cap = sms * LzCfg<2>::MIN_CTAS, g1 = cap < m ? cap : m;
                b2c_lz_parse2_kernel<<<g1, LzCfg<2>::NT, LzLayout<2>::SMEM_BYTES, st>>>(P);
            } else {
                const unsigned cap = sms * LzCfg<5>::MIN_CTAS, g1 = cap < m ? cap : m;
                b2c_lz_parse3_kernel<<<g1, LzCfg<5>::NT, LzLayout<5>::SMEM_BYTES, st>>>(P);
            }
            PEV(2);
            const unsigned gh = sms * HIST_CTAS_PER_SM < m ? sms * HIST_CTAS_PER_SM : m;
            b2c_zstd_hist_kernel<<<gh, HIST_NT, HIST_SMEM_BYTES, st>>>(P);
            ctx->launches += 2;
        }
        PEV(3);
        const unsigned m2 = (m + TABLES_NW - 1) / TABLES_NW;     // K2 takes one chunk per warp at a time
        const unsigned g2 = sms * TABLES_CTAS_PER_SM < m2 ? sms * TABLES_CTAS_PER_SM : m2;
        b2c_zstd_tables_kernel<<<g2, TABLES_NT, 0, st>>>(P);
        PEV(4);
        b2c_zstd_chains_kernel<<<(m + 31) / 32, CHAIN_NT + ((wantXxh && ctx->enc_fused_xxh) ? CHAIN_XXH_NT : 0), CHAIN_SMEM_BYTES, st>>>(P);
        PEV(5);
        if (blockmax > 65536) b2c_zstd_pack128_kernel<<<m, PACK_NT, PackCfg<131072>::SMEM_BYTES, st>>>(P);
        else b2c_zstd_pack_kernel<<<m, PACK_NT, PACK_SMEM_BYTES, st>>>(P);
        PEV(6);
#undef PEV
        ctx->launches += 3;
        CK(cudaGetLastError());
    }
    return ctx_order_end(ctx, st);
}

int b2c_zstd_encode_device(b2c_ctx *ctx, int level, int flags, const void *d_src, size_t src_stride,
                           const uint32_t *d_sizes, uint32_t size_all, void *d_dst, size_t dst_stride,
                           int64_t *d_out_sizes, uint32_t nchunks, void *stream) {
    return launch_encode(ctx, level, flags, d_src, src_stride, d_sizes, size_all, d_dst, dst_stride, d_out_sizes,
                         nchunks, nullptr, nullptr, nullptr, 0, (cudaStream_t)stream);
}

int b2c_zstd_encode_device_debug(b2c_ctx *ctx, int level, int flags, const void *d_src, size_t src_stride,
                                 const uint32_t *d_sizes, uint32_t size_all, void *d_dst, size_t dst_stride,
                                 int64_t *d_out_sizes, uint32_t nchunks, uint32_t *d_dbg_hdr, uint32_t *d_dbg_seqs,
                                 uint8_t *d_dbg_lits, uint32_t dbg_seq_cap, void *stream) {
    return launch_encode(ctx, level, flags, d_src, src_stride, d_sizes, size_all, d_dst, dst_stride,
                         d_out_sizes, nchunks, d_dbg_hdr, d_dbg_seqs, d_dbg_lits, dbg_seq_cap, (cudaStream_t)stream);
}

int b2c_zstd_encode_device_timed(b2c_ctx *ctx, int flags, const void *d_src, size_t src_stride, uint32_t size_all,
                                 void *d_dst, size_t dst_stride, int64_t *d_out_sizes, uint32_t nchunks,
                                 unsigned long long *d_cycles, void *stream) {
    return launch_encode(ctx, B2C_LEVEL_FASTEST, flags, d_src, src_stride, nullptr, size_all, d_dst, dst_stride,
                         d_out_sizes, nchunks, nullptr, nullptr, nullptr, 0, (cudaStream_t)stream, d_cycles);
}


// ------------------------------------------------------------------------------------------------ frame mode
// zstd.Encoder.EncodeAll of an input larger than one block (zstd/encoder.go:796-830): ONE frame per input -- header with
// the content size, the blocks, the XXH64 of the whole content.  Every block is encoded by the same six-kernel pipeline
// as an independent chunk, with two differences: the match finder sees the `hist` bytes before the block (previous
// blocks of the same frame, already in memory), and the blocks are bare (no frame header / checksum of their own).
// Blocks are entropy-coded independently (no repeat-mode tables between blocks, which would serialise a frame's
// blocks; the reference's seqCoders.setPrev / compModeRepeat, zstd/seqenc.go:19-42, is a size optimisation only).
// XXH64 of every frame's content: one warp per frame (xxh64_warp: the warp streams, four lanes hash)
constexpr int FRAME_XXH_WARPS = 4;
__global__ void __launch_bounds__(FRAME_XXH_WARPS * 32) b2c_zstd_frame_xxh_kernel(const uint8_t *src, const FrameDesc *fr, uint64_t *xxh, uint32_t nframes) {
    __shared__ __align__(16) uint8_t stg[FRAME_XXH_WARPS][2 * XXH_TILE];
    const unsigned w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t f = blockIdx.x * FRAME_XXH_WARPS + w;
    if (f >= nframes || !fr[f].crc) return;
    const uint64_t h = xxh64_warp(src + fr[f].off, fr[f].size, stg[w], lane);
    if (lane == 0) xxh[f] = h;
}
// base[k + 1] = base[k] + bytes of sub-batch k (offsets[m] = total of the scan)
__global__ void b2c_frame_base_kernel(uint64_t *base, uint32_t k, const uint64_t *offsets, uint32_t m) { base[k + 1] = base[k] + offsets[m]; }
__global__ void b2c_frame_place_kernel(const uint8_t *slots, uint64_t slot_stride, const int64_t *sizes, const uint64_t *offsets,
                                       const uint64_t *base, uint32_t k, const EncBlockDesc *desc, const FrameDesc *fr,
                                       uint8_t *packed, uint64_t cap, uint64_t *pos, uint32_t c0, uint32_t m) {
    for (uint32_t c = blockIdx.x; c < m; c += gridDim.x)
        frame_place_block(slots, slot_stride, sizes, offsets, base[k], desc, fr, packed, cap, pos, c0, c, threadIdx.x, blockDim.x);
}
__global__ void b2c_frame_finish_kernel(const FrameDesc *fr, const uint64_t *pos, const int64_t *sizes_all, const uint64_t *xxh,
                                        uint8_t *packed, uint64_t cap, uint64_t *out_offsets, int64_t *out_sizes, uint32_t nframes) {
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f < nframes) frame_finish_one(fr, pos, sizes_all, xxh, packed, cap, out_offsets, out_sizes, f);
}

__global__ void b2c_s2_stream_total_kernel(const uint64_t *base, uint32_t nsub, uint64_t *total) { *total = 10 + base[nsub]; }

size_t b2c_zstd_frame_bound(size_t size, int level) {
    if (!level_ok(level)) return 0;
    const FrameGeom g = frame_geom(level);
    const size_t blocks = size ? (size + g.block - 1) / g.block : 1;
    return 14 + 4 + 3 * blocks + size;        // maxHeaderSize + checksum + one block header per block (raw blocks at worst)
}

// Device-resident frame mode.  Frame f = h_src_sizes[f] bytes at d_src + h_src_offsets[f] (host arrays: the block list is
// planned on the host).  Frames are written back to back into d_dst (capacity dst_cap); d_dst_offsets[f] / d_out_sizes[f]
// (device arrays) receive where frame f starts and its size (negative = error).  Asynchronous on `stream`.
int b2c_zstd_encode_frames_device(b2c_ctx *ctx, int level, int flags, const void *d_src, const uint64_t *h_src_offsets,
                                  const uint64_t *h_src_sizes, uint32_t nframes, void *d_dst, uint64_t dst_cap,
                                  uint64_t *d_dst_offsets, int64_t *d_out_sizes, void *stream) {
    if (!ctx) return B2C_ERR_NO_DEVICE;
    if (!level_ok(level)) return B2C_ERR_UNSUPPORTED;
    if (nframes == 0) return B2C_OK;
    if (!h_src_offsets || !h_src_sizes || !d_dst_offsets || !d_out_sizes) return B2C_ERR_ARG;
    CK(cudaSetDevice(ctx->device));
    cudaStream_t st = (cudaStream_t)stream;
    const FrameGeom g = frame_geom(level);
    const bool crc = (flags & B2C_ZSTD_CRC) != 0;
    // ---- plan: block list and frame table
    std::vector<EncBlockDesc> blocks;
    std::vector<FrameDesc> frames;
    if (!frame_plan(level, crc, h_src_offsets, h_src_sizes, nframes, blocks, frames)) return B2C_ERR_ARG;
    const uint32_t nblocks = (uint32_t)blocks.size();
    const uint32_t subMax = level_block(level) > 65536 ? 4096u : 8192u;
    const uint32_t sub = nblocks < subMax ? nblocks : subMax, nsub = (nblocks + sub - 1) / sub;
    const size_t slotB = (size_t)g.block + 512;
    // ---- device memory of the call: descriptors | frame table | per-block sizes, positions | scan offsets | bases | xxh | slots
    Layout L;
    const size_t oDesc = L.take(sizeof(EncBlockDesc) * nblocks), oFr = L.take(sizeof(FrameDesc) * nframes),
                 oSizes = L.take(sizeof(int64_t) * nblocks), oPos = L.take(sizeof(uint64_t) * nblocks),
                 oScan = L.take(sizeof(uint64_t) * ((size_t)sub + 1)), oBase = L.take(sizeof(uint64_t) * ((size_t)nsub + 1)),
                 oXxh = L.take(sizeof(uint64_t) * nframes), oSlots = L.take(slotB * sub);
    { int r = reserve(ctx, ctx->d_fr, L.end); if (r) return r; }
    { int r = ctx_order_begin(ctx, st); if (r) return r; }   // (the frame buffers belong to the context like the work pool)
    const Buf<> &B = ctx->d_fr;
    EncBlockDesc *d_desc = B.at<EncBlockDesc>(oDesc);
    FrameDesc *d_frames = B.at<FrameDesc>(oFr);
    int64_t *d_sizes = B.at<int64_t>(oSizes);
    uint64_t *d_pos = B.at<uint64_t>(oPos), *d_scan = B.at<uint64_t>(oScan), *d_base = B.at<uint64_t>(oBase),
             *d_xxh = B.at<uint64_t>(oXxh);
    uint8_t *d_slots = B.at<uint8_t>(oSlots);
    // pageable host vectors: the copies complete before cudaMemcpyAsync returns (staged by the runtime)
    CK(cudaMemcpyAsync(d_desc, blocks.data(), sizeof(EncBlockDesc) * nblocks, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(d_frames, frames.data(), sizeof(FrameDesc) * nframes, cudaMemcpyHostToDevice, st));
    CK(cudaMemsetAsync(d_base, 0, sizeof(uint64_t), st));
    if (crc) {
        b2c_zstd_frame_xxh_kernel<<<(nframes + FRAME_XXH_WARPS - 1) / FRAME_XXH_WARPS, FRAME_XXH_WARPS * 32, 0, st>>>(
            (const uint8_t *)d_src, d_frames, d_xxh, nframes);
        ctx->launches += 1;
    }
    for (uint32_t k = 0; k < nsub; k++) {
        const uint32_t c0 = k * sub, m = (nblocks - c0 < sub) ? nblocks - c0 : sub;
        int r = launch_encode(ctx, level, 0, d_src, 0, nullptr, 0, d_slots, slotB, d_sizes + c0, m, nullptr, nullptr, nullptr, 0,
                              st, nullptr, 0, d_desc + c0);
        if (r) return r;
        b2c_scan_sizes_kernel<<<1, 1024, 0, st>>>(d_sizes + c0, d_scan, m);
        b2c_frame_base_kernel<<<1, 1, 0, st>>>(d_base, k, d_scan, m);
        b2c_frame_place_kernel<<<(unsigned)ctx->sm_count * 8, 256, 0, st>>>(d_slots, slotB, d_sizes + c0, d_scan, d_base, k, d_desc,
                                                                              d_frames, (uint8_t *)d_dst, dst_cap, d_pos, c0, m);
        ctx->launches += 3;
    }
    b2c_frame_finish_kernel<<<(nframes + 127) / 128, 128, 0, st>>>(d_frames, d_pos, d_sizes, d_xxh, (uint8_t *)d_dst, dst_cap,
                                                                    d_dst_offsets, d_out_sizes, nframes);
    ctx->launches += 1;
    CK(cudaGetLastError());
    return ctx_order_end(ctx, st);
}

// Host-buffer frame mode: what a cgo shim calls for EncodeAll(src) with len(src) > one block (any mix of sizes).
// srcs[i] -> one frame in dsts[i] (capacity dst_caps[i] >= b2c_zstd_frame_bound); sizes_out[i] = frame bytes or a negative error.
int b2c_zstd_encode_frames(b2c_ctx *ctx, int level, int flags, const void *const *srcs, const size_t *src_sizes,
                           void *const *dsts, const size_t *dst_caps, int64_t *sizes_out, size_t n) {
    if (!ctx) return B2C_ERR_NO_DEVICE;
    if (!level_ok(level)) return B2C_ERR_UNSUPPORTED;
    if (n == 0) return B2C_OK;
    if (n > 0x7fffffffull) return B2C_ERR_ARG;
    CK(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    std::vector<uint64_t> offs(n), lens(n);
    uint64_t tin = 0, tout = 0;
    for (size_t i = 0; i < n; i++) {
        offs[i] = tin; lens[i] = src_sizes[i];
        tin += (src_sizes[i] + 15) & ~(uint64_t)15;          // frames start 16-byte aligned (bulk-copy staging of their blocks)
        tout += b2c_zstd_frame_bound(src_sizes[i], level);
    }
    const size_t inB = tin + 64, outB = tout + 64, metaB = (sizeof(uint64_t) + sizeof(int64_t)) * n;
    Layout L;
    const size_t oIn = L.take(inB), oOut = L.take(outB), oMeta = L.take(metaB);   // meta: frame offsets | frame sizes
    { int r = reserve(ctx, ctx->d_fr_io, inB + outB + metaB + 512); if (r) return r; }   // (512: the rounding of in and out)
    uint8_t *d_in = ctx->d_fr_io.at<uint8_t>(oIn), *d_out = ctx->d_fr_io.at<uint8_t>(oOut);
    uint64_t *d_off = ctx->d_fr_io.at<uint64_t>(oMeta);
    int64_t *d_sz = (int64_t *)(d_off + n);
    for (size_t i = 0; i < n; i++)
        if (src_sizes[i]) CK(cudaMemcpyAsync(d_in + offs[i], srcs[i], src_sizes[i], cudaMemcpyHostToDevice, st));
    int r = b2c_zstd_encode_frames_device(ctx, level, flags, d_in, offs.data(), lens.data(), (uint32_t)n, d_out, outB, d_off, d_sz, st);
    if (r) { cudaStreamSynchronize(st); return r; }
    std::vector<uint64_t> ho(n);
    std::vector<int64_t> hs(n);
    CK(cudaMemcpyAsync(ho.data(), d_off, sizeof(uint64_t) * n, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(hs.data(), d_sz, sizeof(int64_t) * n, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    for (size_t i = 0; i < n; i++) {
        if (hs[i] > 0 && (size_t)hs[i] > dst_caps[i]) hs[i] = B2C_ERR_DST_SMALL;
        if (hs[i] > 0) CK(cudaMemcpyAsync(dsts[i], d_out + ho[i], (size_t)hs[i], cudaMemcpyDeviceToHost, st));
        sizes_out[i] = hs[i];
    }
    CK(cudaStreamSynchronize(st));
    return B2C_OK;
}

int b2c_zstd_encode_chunks(b2c_ctx *ctx, int level, int flags, const void *const *srcs, const size_t *src_sizes,
                           void *const *dsts, const size_t *dst_caps, int64_t *sizes_out, size_t n) {
    if (!ctx) return B2C_ERR_NO_DEVICE;
    if (!level_ok(level)) return B2C_ERR_UNSUPPORTED;
    if (!ctx->max_chunks) return B2C_ERR_ARG;
    const size_t blk = level_block(level), slotB = level_slot(level);
    const size_t mcap = ctx->max_chunks * (size_t)ENC_MAX_CHUNK / blk;   // the staging buffers hold max_chunks x 64 KiB
    if (!mcap) return B2C_ERR_ARG;
    CK(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    EncSlot &S = ctx->slot[0];
    for (size_t base = 0; base < n; base += mcap) {
        size_t m = n - base;
        if (m > mcap) m = mcap;
        // contiguous equal-sized input needs no host-side staging copy
        bool contiguous = true;
        for (size_t i = 0; i < m; i++) {
            if (src_sizes[base + i] > blk) { contiguous = false; }
            if (i + 1 < m && ((const uint8_t *)srcs[base + i] + src_sizes[base + i] != (const uint8_t *)srcs[base + i + 1] ||
                              src_sizes[base + i] != blk))
                contiguous = false;
            S.h_src_sizes.p[i] = (uint32_t)(src_sizes[base + i] > blk ? blk + 1 : src_sizes[base + i]);
        }
        size_t in_bytes = 0;
        for (size_t i = 0; i < m; i++) in_bytes += src_sizes[base + i];
        if (contiguous) {
            CK(cudaMemcpyAsync(S.d_in.p, srcs[base], in_bytes, cudaMemcpyHostToDevice, st));
        } else {
            {
                uint8_t *hin = S.h_in.p;
                parallel_pieces(m, in_bytes, [=](size_t i) {
                    const size_t sz = src_sizes[base + i] > blk ? 0 : src_sizes[base + i];
                    memcpy(hin + i * (size_t)blk, srcs[base + i], sz);
                });
            }
            CK(cudaMemcpyAsync(S.d_in.p, S.h_in.p, m * (size_t)blk, cudaMemcpyHostToDevice, st));
        }
        CK(cudaMemcpyAsync(S.d_src_sizes.p, S.h_src_sizes.p, m * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
        int rc = launch_encode(ctx, level, flags, S.d_in.p, blk, S.d_src_sizes.p, 0, S.d_out.p, slotB,
                               S.d_sizes.p, (uint32_t)m, nullptr, nullptr, nullptr, 0, st);
        if (rc) return rc;
        b2c_scan_sizes_kernel<<<1, 1024, 0, st>>>(S.d_sizes.p, S.d_offsets.p, (uint32_t)m);
        b2c_pack_kernel<<<ctx->sm_count * 4, 256, 0, st>>>(S.d_out.p, slotB, S.d_sizes.p, S.d_offsets.p, S.d_packed.p, (uint32_t)m);
        ctx->launches += 2;
        int64_t *h_sz = S.h_sizes.p;
        uint64_t *h_off = reinterpret_cast<uint64_t *>(h_sz + m);
        CK(cudaMemcpyAsync(h_sz, S.d_sizes.p, m * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(h_off, S.d_offsets.p, (m + 1) * sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        uint64_t total = h_off[m];
        CK(cudaMemcpyAsync(S.h_out.p, S.d_packed.p, total, cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        {
            const uint8_t *hout = S.h_out.p;
            parallel_pieces(m, (size_t)total, [=](size_t i) {
                int64_t sz = h_sz[i];
                if (sz > 0 && (size_t)sz > dst_caps[base + i]) sz = B2C_ERR_DST_SMALL;
                if (sz > 0) memcpy(dsts[base + i], hout + h_off[i], (size_t)sz);
                sizes_out[base + i] = sz;
            });
        }
    }
    return B2C_OK;
}



// ---- host-side helpers of the host-buffer calls ---------------------------------------------------------------
// A Go caller's slices are ordinary (pageable) memory: a cudaMemcpyAsync from them is staged by the driver through a
// small pinned window and blocks.  The packed call therefore stages pageable buffers itself: several host threads copy
// into / out of the context's pinned buffers while the copy engines and kernels work on the neighbouring batches.
static bool host_ptr_is_pinned(const void *p) {
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
    return a.type == cudaMemoryTypeHost || a.type == cudaMemoryTypeManaged;
}
static void parallel_memcpy(void *dst, const void *src, size_t bytes) {
    const size_t kMin = 4u << 20;
    unsigned hw = std::thread::hardware_concurrency();
    unsigned nt = hw ? (hw < 8 ? hw : 8) : 4;
    if (bytes < 2 * kMin || nt < 2) { memcpy(dst, src, bytes); return; }
    if ((size_t)nt * kMin > bytes) nt = (unsigned)(bytes / kMin);
    const size_t per = ((bytes / nt) + 4095) & ~(size_t)4095;
    std::vector<std::thread> th;
    for (unsigned t = 1; t < nt; t++) {
        const size_t lo = (size_t)t * per;
        if (lo >= bytes) break;
        const size_t len = (lo + per <= bytes && t + 1 < nt) ? per : bytes - lo;
        th.emplace_back([=]() { memcpy((uint8_t *)dst + lo, (const uint8_t *)src + lo, len); });
    }
    memcpy(dst, src, per < bytes ? per : bytes);
    for (auto &x : th) x.join();
}

// Contiguous host input -> packed host output (concatenated frames).  Three streams (H2D, kernels, D2H) and two
// buffer slots: the H2D copy of batch b+1 and the D2H copy of batch b-1 overlap the kernels of batch b.  This is the
// shape of a large EncodeAll / of a WithConcurrentBlocks job (zstd/enc_jobs.go): the caller gets one valid zstd
// stream plus the per-chunk frame table.  h_src / h_dst should be pinned (cudaHostRegister / torch pin_memory)
// for full PCIe rate; pageable memory works but is staged by the driver.
static int encode_packed_impl(b2c_ctx *ctx, int level, int flags, const void *h_src, size_t src_bytes,
                              uint32_t chunk_size, void *h_dst, size_t dst_cap, int64_t *sizes_out,
                              uint64_t *offsets_out, size_t *total_out) {
    if (!ctx) return B2C_ERR_NO_DEVICE;
    if (!level_ok(level)) return B2C_ERR_UNSUPPORTED;
    const size_t blk = level_block(level), slotB = level_slot(level);
    if (!ctx->max_chunks || chunk_size == 0 || chunk_size > blk) return B2C_ERR_ARG;
    CK(cudaSetDevice(ctx->device));
    const size_t nchunks = src_bytes == 0 ? 1 : (src_bytes + chunk_size - 1) / chunk_size;
    const size_t B = ctx->max_chunks * (size_t)ENC_MAX_CHUNK / blk;   // the staging buffers hold max_chunks x 64 KiB
    if (!B) return B2C_ERR_ARG;
    // Batch schedule: full batches, then a tail that halves down to about four chunks per SM.  The H2D stream is the
    // bottleneck of the pipeline, so the time after the last H2D copy (kernels + D2H of the last batch) is pure
    // overhead; a small last batch keeps it short.
    std::vector<size_t> bstart, bcount;
    {
        size_t c0 = 0, rem = nchunks;
        // (below about four chunks per SM a batch is bound by the latency of its serial kernels, not by its size)
        const size_t floorB = (size_t)ctx->sm_count * 4 < B ? (size_t)ctx->sm_count * 4 : B;
        while (rem > 0) {
            size_t m;
            if (rem > B) m = B;
            else if (rem > 2 * floorB) m = rem / 2;
            else m = rem;
            bstart.push_back(c0); bcount.push_back(m);
            c0 += m; rem -= m;
        }
    }
    const size_t nb = bcount.size();
    cudaStream_t st_c = ctx->stream, st_in = ctx->stream2, st_out = ctx->stream3;
    // pageable caller memory is staged through the context's pinned buffers (see parallel_memcpy above)
    const bool stage_in = src_bytes > 0 && !host_ptr_is_pinned(h_src);
    const bool stage_out = !host_ptr_is_pinned(h_dst);
    if (stage_in || stage_out) {
        { int r = reserve(ctx, ctx->slot[1].h_in, ctx->max_chunks * (size_t)ENC_MAX_CHUNK); if (r) return r; }
        { int r = reserve(ctx, ctx->slot[1].h_out, ctx->max_chunks * (size_t)kSlot); if (r) return r; }
    }
    struct Pending { bool live; uint64_t pos, bytes; } pend[2] = {{false, 0, 0}, {false, 0, 0}};
    // a staged D2H copy of slot sl has landed in pinned memory: hand it to the caller's buffer
    auto drain = [&](int sl) -> int {
        if (!pend[sl].live) return B2C_OK;
        if (cudaEventSynchronize(ctx->slot[sl].ev_out) != cudaSuccess) return B2C_ERR_CUDA;
        parallel_memcpy((uint8_t *)h_dst + pend[sl].pos, ctx->slot[sl].h_out.p, pend[sl].bytes);
        pend[sl].live = false;
        return B2C_OK;
    };
    uint64_t out_pos = 0;
    int rc = B2C_OK;
    // batch b's kernels are done: place its frames in the output stream and start the D2H copy
    auto finish = [&](size_t b) -> int {
        const int sl = (int)(b & 1);
        EncSlot &S = ctx->slot[sl];
        size_t c0 = bstart[b], m = bcount[b];
        if (cudaEventSynchronize(S.ev) != cudaSuccess) return B2C_ERR_CUDA;
        const int64_t *h_sz = S.h_sizes.p;
        const uint64_t *h_off = reinterpret_cast<const uint64_t *>(h_sz + m);
        uint64_t total = h_off[m];
        if (out_pos + total > dst_cap) return B2C_ERR_DST_SMALL;
        if (stage_out) {
            { int rd = drain(sl); if (rd) return rd; }            // the slot's pinned buffer still holds batch b-2
            if (cudaMemcpyAsync(S.h_out.p, S.d_packed.p, total, cudaMemcpyDeviceToHost, st_out) != cudaSuccess) return B2C_ERR_CUDA;
            pend[sl].live = true; pend[sl].pos = out_pos; pend[sl].bytes = total;
        } else if (cudaMemcpyAsync((uint8_t *)h_dst + out_pos, S.d_packed.p, total, cudaMemcpyDeviceToHost, st_out) != cudaSuccess)
            return B2C_ERR_CUDA;
        if (cudaEventRecord(S.ev_out, st_out) != cudaSuccess) return B2C_ERR_CUDA;
        if (stage_out) { int rd = drain(sl ^ 1); if (rd) return rd; }   // batch b-1's bytes have had a whole batch to arrive
        for (size_t i = 0; i < m; i++) {
            sizes_out[c0 + i] = h_sz[i];
            if (offsets_out) offsets_out[c0 + i] = out_pos + h_off[i];
            if (h_sz[i] < 0) rc = (int)h_sz[i];
        }
        out_pos += total;
        return B2C_OK;
    };
    // H2D of batch b into its slot; the slot's input buffer is free once the kernels of batch b-2 have run
    std::vector<const uint32_t *> bss(nb, nullptr);
    auto upload = [&](size_t b) -> int {
        const int sl = (int)(b & 1);
        EncSlot &S = ctx->slot[sl];
        size_t c0 = bstart[b], m = bcount[b];
        size_t off = c0 * (size_t)chunk_size;
        size_t bytes = (off + m * (size_t)chunk_size <= src_bytes) ? m * (size_t)chunk_size : src_bytes - off;
        if (b >= 2) CK(cudaStreamWaitEvent(st_in, S.ev, 0));
        const uint8_t *from = (const uint8_t *)h_src + off;
        if (stage_in && bytes) {
            if (b >= 2) CK(cudaEventSynchronize(S.ev_in));      // the H2D copy of batch b-2 has left the pinned buffer
            parallel_memcpy(S.h_in.p, from, bytes);
            from = S.h_in.p;
        }
        if (bytes) CK(cudaMemcpyAsync(S.d_in.p, from, bytes, cudaMemcpyHostToDevice, st_in));
        if (bytes != m * (size_t)chunk_size) {  // ragged last chunk (or empty input): explicit sizes
            for (size_t i = 0; i < m; i++) {
                size_t o = i * (size_t)chunk_size;
                S.h_src_sizes.p[i] = (uint32_t)(o >= bytes ? 0 : (bytes - o < chunk_size ? bytes - o : chunk_size));
            }
            CK(cudaMemcpyAsync(S.d_src_sizes.p, S.h_src_sizes.p, m * sizeof(uint32_t), cudaMemcpyHostToDevice, st_in));
            bss[b] = S.d_src_sizes.p;
        }
        CK(cudaEventRecord(S.ev_in, st_in));
        return B2C_OK;
    };
    // The copy of batch b+2 is queued before the host waits for batch b-1, so the H2D engine (the bottleneck) always
    // has the next copy in its queue.
    { int r0 = upload(0); if (r0) return r0; }
    if (nb > 1) { int r1 = upload(1); if (r1) return r1; }
    for (size_t b = 0; b < nb; b++) {
        const int sl = (int)(b & 1);
        EncSlot &S = ctx->slot[sl];
        size_t m = bcount[b];
        // kernels: need the input; the packed-output slot is free once batch b-2's D2H copy is done
        CK(cudaStreamWaitEvent(st_c, S.ev_in, 0));
        if (b >= 2) CK(cudaStreamWaitEvent(st_c, S.ev_out, 0));
        int r = launch_encode(ctx, level, flags, S.d_in.p, chunk_size, bss[b], chunk_size, S.d_out.p, slotB, S.d_sizes.p,
                              (uint32_t)m, nullptr, nullptr, nullptr, 0, st_c, nullptr, sl);
        if (r) return r;
        b2c_scan_sizes_kernel<<<1, 1024, 0, st_c>>>(S.d_sizes.p, S.d_offsets.p, (uint32_t)m);
        b2c_pack_kernel<<<ctx->sm_count * 4, 256, 0, st_c>>>(S.d_out.p, slotB, S.d_sizes.p, S.d_offsets.p, S.d_packed.p, (uint32_t)m);
        ctx->launches += 2;
        CK(cudaMemcpyAsync(S.h_sizes.p, S.d_sizes.p, m * sizeof(int64_t), cudaMemcpyDeviceToHost, st_c));
        CK(cudaMemcpyAsync(S.h_sizes.p + m, S.d_offsets.p, (m + 1) * sizeof(uint64_t), cudaMemcpyDeviceToHost, st_c));
        CK(cudaEventRecord(S.ev, st_c));
        if (b + 2 < nb) { int r3 = upload(b + 2); if (r3) return r3; }
        if (b >= 1) { int r2 = finish(b - 1); if (r2) return r2; }
    }
    { int r2 = finish(nb - 1); if (r2) return r2; }
    CK(cudaStreamSynchronize(st_in));
    CK(cudaStreamSynchronize(st_c));
    CK(cudaStreamSynchronize(st_out));
    { int rd = drain(0); if (rd) return rd; }
    { int rd = drain(1); if (rd) return rd; }
    if (total_out) *total_out = out_pos;
    return rc;
}

int b2c_zstd_encode_packed(b2c_ctx *ctx, int level, int flags, const void *h_src, size_t src_bytes,
                           uint32_t chunk_size, void *h_dst, size_t dst_cap, int64_t *sizes_out,
                           uint64_t *offsets_out, size_t *total_out) {
    const int rc = encode_packed_impl(ctx, level, flags, h_src, src_bytes, chunk_size, h_dst, dst_cap, sizes_out, offsets_out,
                                      total_out);
    if (rc != B2C_OK && ctx && ctx->stream) {
        // an error return must not leave copies in flight that read h_src / write h_dst, nor the slots mid-pipeline
        cudaStreamSynchronize(ctx->stream2);
        cudaStreamSynchronize(ctx->stream);
        cudaStreamSynchronize(ctx->stream3);
    }
    return rc;
}

// ---- decoder ------------------------------------------------------------------------------------
// Pointer-table calls: n separately allocated host pieces <-> one packed device range.  Thousands of small
// cudaMemcpyAsync calls cost more than the bytes they move (and block on pageable memory), so the pieces are gathered
// into / scattered from one pinned staging buffer and cross the bus as ONE copy each way.  offs[i] = offset of piece i in
// the device range `d_base[0, total)`.
static const size_t kStageLimit = (size_t)1 << 30;
static int gather_h2d(b2c_ctx *ctx, const void *const *srcs, const size_t *sizes, const uint64_t *offs, size_t n, uint8_t *d_base,
                      size_t total, cudaStream_t st) {
    if (total == 0) return B2C_OK;
    if (total > kStageLimit) {
        for (size_t i = 0; i < n; i++)
            if (sizes[i]) CK(cudaMemcpyAsync(d_base + offs[i], srcs[i], sizes[i], cudaMemcpyHostToDevice, st));
        return B2C_OK;
    }
    int rc = reserve(ctx, ctx->h_stg_in, total);
    if (rc) return rc;
    {
        uint8_t *stg = ctx->h_stg_in.p;
        parallel_pieces(n, total, [=](size_t i) { if (sizes[i]) memcpy(stg + offs[i], srcs[i], sizes[i]); });
    }
    CK(cudaMemcpyAsync(d_base, ctx->h_stg_in.p, total, cudaMemcpyHostToDevice, st));
    return B2C_OK;
}
// results: piece i = d_base[offs[i], offs[i] + lens[i]) -> dsts[i]; synchronises the stream
static int scatter_d2h(b2c_ctx *ctx, void *const *dsts, const size_t *lens, const uint64_t *offs, size_t n, const uint8_t *d_base,
                       size_t range, cudaStream_t st) {
    size_t useful = 0;
    for (size_t i = 0; i < n; i++) useful += lens[i];
    if (useful == 0) { CK(cudaStreamSynchronize(st)); return B2C_OK; }
    if (range > kStageLimit || useful * 2 < range) {          // sparse or huge: copy the pieces
        for (size_t i = 0; i < n; i++)
            if (lens[i]) CK(cudaMemcpyAsync(dsts[i], d_base + offs[i], lens[i], cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        return B2C_OK;
    }
    int rc = reserve(ctx, ctx->h_stg_out, range);
    if (rc) return rc;
    CK(cudaMemcpyAsync(ctx->h_stg_out.p, d_base, range, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    {
        const uint8_t *stg = ctx->h_stg_out.p;
        parallel_pieces(n, useful, [=](size_t i) { if (lens[i]) memcpy(dsts[i], stg + offs[i], lens[i]); });
    }
    return B2C_OK;
}

}  // extern "C": HostBatch has member templates

static uint32_t clamp32(size_t v) { return (uint32_t)(v > 0xffffffffull ? 0xffffffffull : v); }

// One pointer-table batch: n caller pieces, their inputs placed in d_dec_in and their outputs in d_dec_out, and m device
// items whose per-item arrays -- with the extra arrays a call lists -- form one layout that crosses to d_dec_meta in one
// copy.  m == n except in zstd decode, whose items are frames.  Use: check(), place() / place_items(), stage_in(), the
// launch, results(), scatter().
struct HostBatch {
    struct Arrays { uint64_t *src_off, *dst_off; int64_t *res; uint32_t *src_sizes, *dst_caps; };
    b2c_ctx *ctx;
    size_t n, m;
    std::vector<uint64_t> in_off, out_off;      // piece i's offset in d_dec_in / d_dec_out
    uint64_t in_bytes = 0, out_bytes = 0;
    Layout L;
    size_t off[5];
    std::vector<size_t> ex;                     // offsets of the extra arrays, in the order given
    std::vector<uint8_t> host;                  // the arrays and the extras; regions L takes later are device-only
    Arrays h, d = {};                           // in `host` / in d_dec_meta (set by stage_in)

    HostBatch(b2c_ctx *c, size_t n_, size_t m_, std::initializer_list<size_t> extra = {})
        : ctx(c), n(n_), m(m_), in_off(n_), out_off(n_) {
        off[0] = L.take(sizeof(uint64_t) * m); off[1] = L.take(sizeof(uint64_t) * m); off[2] = L.take(sizeof(int64_t) * m);
        off[3] = L.take(sizeof(uint32_t) * m); off[4] = L.take(sizeof(uint32_t) * m);
        for (size_t b : extra) ex.push_back(L.take(b));
        host.resize(L.end);
        h = at(host.data());
    }
    // The checks every pointer-table call makes after its own: the item count, then each input against the call's limit.
    static int check(b2c_ctx *ctx, size_t n, const size_t *src_sizes, size_t limit) {
        if (n > 0xffffffffull) return B2C_ERR_ARG;
        CK(cudaSetDevice(ctx->device));
        for (size_t i = 0; i < n; i++)
            if (src_sizes[i] > limit) return B2C_ERR_ARG;
        return B2C_OK;
    }
    Arrays at(uint8_t *base) const {
        return {reinterpret_cast<uint64_t *>(base + off[0]), reinterpret_cast<uint64_t *>(base + off[1]),
                reinterpret_cast<int64_t *>(base + off[2]), reinterpret_cast<uint32_t *>(base + off[3]),
                reinterpret_cast<uint32_t *>(base + off[4])};
    }
    template <class T> T *h_at(size_t o) { return reinterpret_cast<T *>(host.data() + o); }
    template <class T> T *d_at(size_t o) const { return ctx->d_dec_meta.at<T>(o); }
    // Piece i's input and output offsets: packed at 16-byte alignment (stride 0) or at a fixed stride.
    void place(const size_t *in_len, size_t in_stride, const size_t *out_len, size_t out_stride) {
        for (size_t i = 0; i < n; i++) {
            in_off[i] = in_bytes; out_off[i] = out_bytes;
            in_bytes += in_stride ? in_stride : (in_len[i] + 15) & ~(uint64_t)15;
            out_bytes += out_stride ? out_stride : ((uint64_t)clamp32(out_len[i]) + 15) & ~(uint64_t)15;
        }
    }
    // place() with one item per piece: its input, its output and its capacity clamped to 32 bits.
    void place_items(const size_t *src_sizes, size_t in_stride, const size_t *dst_caps, size_t out_stride) {
        place(src_sizes, in_stride, dst_caps, out_stride);
        for (size_t i = 0; i < n; i++) {
            h.src_off[i] = in_off[i]; h.dst_off[i] = out_off[i];
            h.src_sizes[i] = (uint32_t)src_sizes[i]; h.dst_caps[i] = clamp32(dst_caps[i]);
        }
    }
    // Reserves the three buffers, gathers lens[i] bytes of srcs[i] into d_dec_in and uploads the arrays.
    int stage_in(const void *const *srcs, const size_t *lens) {
        int rc;
        if ((rc = reserve(ctx, ctx->d_dec_in, in_bytes + 256))) return rc;
        if ((rc = reserve(ctx, ctx->d_dec_out, out_bytes + 256))) return rc;
        if ((rc = reserve(ctx, ctx->d_dec_meta, L.end + 256))) return rc;
        if ((rc = gather_h2d(ctx, srcs, lens, in_off.data(), n, ctx->d_dec_in.p, in_bytes, ctx->stream))) return rc;
        CK(cudaMemcpyAsync(ctx->d_dec_meta.p, host.data(), host.size(), cudaMemcpyHostToDevice, ctx->stream));
        d = at(ctx->d_dec_meta.p);
        return B2C_OK;
    }
    // A Params struct of a packed call with the batch's buffers and arrays; the rest zeroed.
    template <class P> P params() const {
        P p;
        memset(&p, 0, sizeof(p));
        p.src_base = ctx->d_dec_in.p; p.src_offsets = d.src_off; p.src_sizes = d.src_sizes;
        p.dst_base = ctx->d_dec_out.p; p.dst_offsets = d.dst_off; p.dst_caps = d.dst_caps; p.out_sizes = d.res;
        return p;
    }
    // The m results -> res (host), then synchronises: copies the call enqueued before complete with it.
    int results(int64_t *res) {
        CK(cudaMemcpyAsync(res, d.res, m * sizeof(int64_t), cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        return B2C_OK;
    }
    // A result larger than its piece's capacity becomes B2C_ERR_DST_SMALL; then each positive result's bytes (or, with
    // row, `row` bytes for each result >= 0) go to dsts[i].  Synchronises.
    int scatter(void *const *dsts, int64_t *sizes, const size_t *dst_caps, size_t row = 0) {
        std::vector<size_t> lens(n, 0);
        for (size_t i = 0; i < n; i++) {
            if (sizes[i] > 0 && (size_t)sizes[i] > dst_caps[i]) sizes[i] = B2C_ERR_DST_SMALL;
            if (sizes[i] >= 0) lens[i] = row ? row : (size_t)sizes[i];
        }
        return scatter_d2h(ctx, dsts, lens.data(), out_off.data(), n, ctx->d_dec_out.p, out_bytes, ctx->stream);
    }
};

// Record-bounded launches (LZ4 conversion, inflate): the pass that starts at item c0 takes the items whose records fit
// kRecPassBytes of scratch, at least one.  rec_base (host) holds every item's first record, and the total at [n]; without it
// every item has room for `per` records.  Sets *c1 to the pass's end and returns its record count.
static const uint64_t kRecPassBytes = (uint64_t)4 << 30;
static uint64_t next_pass(uint32_t c0, uint32_t n, const uint64_t *rec_base, uint64_t per, size_t rec_bytes, uint32_t *c1) {
    if (rec_base) {
        uint32_t e = c0 + 1;
        while (e < n && (rec_base[e + 1] - rec_base[c0]) * rec_bytes <= kRecPassBytes) e++;
        *c1 = e;
        return rec_base[e] - rec_base[c0];
    }
    const uint64_t fit = kRecPassBytes / (per * rec_bytes), k = fit > 1 ? fit : 1;
    *c1 = (uint32_t)((uint64_t)c0 + k < n ? c0 + k : n);
    return (uint64_t)(*c1 - c0) * per;
}

extern "C" {

// lit_span: bytes of the output layout (literal areas mirror it: input c's area starts at c * lit_stride, or at
// dst_offsets[c] when lit_stride is 0 -- the caller then guarantees non-overlapping, increasing offsets); 0 = unknown: the
// one-warp decoder takes every input.
static const uint64_t kStagedSpanLimit = 24ull << 30;
// Grid of a one-warp decoder kernel over n inputs (DEC_WARPS per CTA): at most *max_grid CTAs, what the device holds at once.
static unsigned dec_grid(const b2c_ctx *ctx, uint32_t n, unsigned *max_grid = nullptr) {
    const unsigned ctasPerSm = (227u * 1024u) / (DEC_SMEM_BYTES + 1024u);
    const unsigned grid = (n + DEC_WARPS - 1) / DEC_WARPS, maxGrid = (unsigned)ctx->sm_count * (ctasPerSm ? ctasPerSm : 1);
    if (max_grid) *max_grid = maxGrid;
    return grid < maxGrid ? grid : maxGrid;
}
static int launch_decode(b2c_ctx *ctx, ZstdDecParams &P, cudaStream_t st, uint64_t lit_span, uint64_t lit_stride) {
    if (P.nchunks == 0) return B2C_OK;
    unsigned maxGrid;
    const unsigned grid = dec_grid(ctx, P.nchunks, &maxGrid);
    int rc = reserve(ctx, ctx->d_dec_lit, (size_t)maxGrid * DEC_WARPS * DEC_LIT_SCRATCH);
    if (rc) return rc;
    P.lit_scratch = ctx->d_dec_lit.p;
    { int r = ctx_order_begin(ctx, st); if (r) return r; }    // the context's scratch is shared by all streams
    const uint32_t n = P.nchunks;
    const bool prof = ctx->dec_prof != 0;
    // Blocks per input the staged kernels take: FD_MAXB with one lane / quad per input (many inputs), up to FD_MAXB_LONG with one
    // lane / quad per (input, block) when the inputs are few -- then long frames are decoded block-parallel.  The tables are
    // [n][maxb], so n * maxb is bounded.
    uint32_t maxb = FD_MAXB;
    if (n <= 4096) { maxb = (uint32_t)(65536 / n); if (maxb > FD_MAXB_LONG) maxb = FD_MAXB_LONG; }      // (>= 16 blocks per input)
    const bool perBlock = maxb > FD_MAXB;
    const bool staged = ctx->dec_staged && lit_span > 0 && lit_span <= kStagedSpanLimit && (uint64_t)n * maxb * FD_TAB_ENTRIES < (1ull << 31);
    ctx->fd_last = staged;
    if (staged) {
        Layout L;
        const size_t oRec = L.take((size_t)n * sizeof(FdChunk)), oBlk = L.take((size_t)n * maxb * sizeof(FdBlock)),
                     oTab = L.take((size_t)n * maxb * FD_TAB_ENTRIES * sizeof(uint32_t)),
                     oHuf = L.take((size_t)n * maxb * 2048 * sizeof(uint16_t));
        if ((rc = reserve(ctx, ctx->d_fd, L.end))) return rc;
        if ((rc = reserve(ctx, ctx->d_fd_seq, 8 * ((size_t)(lit_span / 3) + 2 * (size_t)n + 8)))) return rc;
        if ((rc = reserve(ctx, ctx->d_fd_lit, (size_t)lit_span + 64))) return rc;
        P.fd = ctx->d_fd.at<FdChunk>(oRec);
        P.fd_blk = ctx->d_fd.at<FdBlock>(oBlk);
        P.fd_maxb = maxb; P.fd_per_block = perBlock ? 1u : 0u;
        P.fd_tabs = ctx->d_fd.at<uint32_t>(oTab);
        P.fd_huf = ctx->d_fd.at<uint16_t>(oHuf);
        P.fd_const = ctx->d_fd_const.p;
        P.fd_seqs = ctx->d_fd_seq.at<uint64_t>(0);
        P.fd_lits = ctx->d_fd_lit.p;
        P.fd_lit_stride = lit_stride;
        const uint32_t units = perBlock ? n * maxb : n;            // what the literal and sequence kernels spread over
        const unsigned groups = (units + FD_LIT_GROUP - 1) / FD_LIT_GROUP;
        if (prof) cudaEventRecord(ctx->dec_ev[0], st);
        b2c_zstd_dec_scan_kernel<<<(n + 31) / 32, 32, 0, st>>>(P);
        if (perBlock) {             // index pass above; now the blocks' contents side by side, then the per-input link pass
            b2c_zstd_dec_scan_block_kernel<<<(units + 31) / 32, 32, 0, st>>>(P);
            b2c_zstd_dec_link_kernel<<<(n + 31) / 32, 32, 0, st>>>(P);
            ctx->launches += 2;
        }
        // the literal kernel and the sequence walk both depend on the scan only and both are bound by the latency of their
        // serial walks, not by any unit: they run side by side (one after the other when per-kernel times are wanted)
        if (prof) {
            cudaEventRecord(ctx->dec_ev[1], st);
            b2c_zstd_dec_lit_kernel<<<(groups + FD_LIT_WARPS - 1) / FD_LIT_WARPS, FD_LIT_WARPS * 32, FD_LIT_WARPS * FD_LIT_WARP_BYTES, st>>>(P);
            cudaEventRecord(ctx->dec_ev[2], st);
            b2c_zstd_dec_seq_kernel<<<(units + 31) / 32, 32, 0, st>>>(P);
        } else {
            // (measured both ways round: the literal kernel on the auxiliary stream is 0.6 ms per GiB better than the sequence
            // walk there; neither order overlaps the two fully -- see DESIGN.md section 3.2 on shared-memory carveouts)
            CK(cudaEventRecord(ctx->dec_fork, st));
            CK(cudaStreamWaitEvent(ctx->dec_aux, ctx->dec_fork, 0));
            b2c_zstd_dec_lit_kernel<<<(groups + FD_LIT_WARPS - 1) / FD_LIT_WARPS, FD_LIT_WARPS * 32, FD_LIT_WARPS * FD_LIT_WARP_BYTES, ctx->dec_aux>>>(P);
            CK(cudaEventRecord(ctx->dec_join, ctx->dec_aux));
            b2c_zstd_dec_seq_kernel<<<(units + 31) / 32, 32, 0, st>>>(P);
            CK(cudaStreamWaitEvent(st, ctx->dec_join, 0));
        }
        if (prof) cudaEventRecord(ctx->dec_ev[3], st);
        b2c_zstd_dec_exec_kernel<<<(n + FD_EXEC_WARPS - 1) / FD_EXEC_WARPS, FD_EXEC_WARPS * 32, 0, st>>>(P);
        if (prof) cudaEventRecord(ctx->dec_ev[4], st);
        if (perBlock) b2c_zstd_dec_xxh_warp_kernel<<<(n + 3) / 4, 128, 0, st>>>(P);     // few, long inputs: a warp streams each
        else b2c_zstd_dec_xxh_kernel<<<(unsigned)(((uint64_t)n * 4 + 127) / 128), 128, 0, st>>>(P);
        if (prof) cudaEventRecord(ctx->dec_ev[5], st);
        ctx->launches += 5;
    }
    b2c_zstd_decode_kernel<<<grid, DEC_WARPS * 32, DEC_SMEM_BYTES, st>>>(P);
    ctx->launches += 1;
    if (prof && staged) {
        cudaEventRecord(ctx->dec_ev[6], st);
        cudaEventSynchronize(ctx->dec_ev[6]);
        for (int i = 0; i < 6; i++) { float ms = 0; cudaEventElapsedTime(&ms, ctx->dec_ev[i], ctx->dec_ev[i + 1]); ctx->dec_ms[i] += ms; }
    }
    CK(cudaGetLastError());
    return ctx_order_end(ctx, st);
}

int b2c_zstd_decode_device(b2c_ctx *ctx, const void *d_src, size_t src_stride, const uint64_t *d_src_offsets,
                           const uint32_t *d_src_sizes, void *d_dst, size_t dst_stride, const uint64_t *d_dst_offsets,
                           uint32_t dst_cap, int64_t *d_out_sizes, uint32_t nchunks, void *stream) {
    if (!ctx) return B2C_ERR_NO_DEVICE;
    if (!d_src_sizes || !d_out_sizes) return B2C_ERR_ARG;
    CK(cudaSetDevice(ctx->device));
    ZstdDecParams P;
    memset(&P, 0, sizeof(P));
    P.src_base = (const uint8_t *)d_src; P.src_stride = src_stride; P.src_offsets = d_src_offsets; P.src_sizes = d_src_sizes;
    P.dst_base = (uint8_t *)d_dst; P.dst_stride = dst_stride; P.dst_offsets = d_dst_offsets; P.dst_cap = dst_cap;
    P.out_sizes = d_out_sizes; P.nchunks = nchunks;
    // literal areas: one of dst_cap bytes per input
    return launch_decode(ctx, P, (cudaStream_t)stream, (uint64_t)nchunks * dst_cap, dst_cap);
}

// Host pre-scan of a zstd stream (no decompression): the frames it is made of, each with its byte range and -- when the
// header carries one -- its Frame_Content_Size.  Header layout as in frameDec.reset (zstd/framedec.go:65-270) /
// Header.Decode (zstd/decodeheader.go:94-229); frame length = header + block headers' sizes (blockdec.go:128-160) +
// checksum.  Returns false when the stream cannot be walked (truncated, bad magic, reserved block type): the caller then
// hands the whole input to one decoder warp, which reports the error the reference reports.
struct FrameSpan { size_t off, len; uint64_t fcs; bool has_fcs, skippable; };
static bool scan_frames(const uint8_t *p, size_t n, std::vector<FrameSpan> &out) {
    size_t pos = 0;
    while (pos < n) {
        if (n - pos < 4) return false;
        const uint32_t magic = (uint32_t)p[pos] | ((uint32_t)p[pos + 1] << 8) | ((uint32_t)p[pos + 2] << 16) | ((uint32_t)p[pos + 3] << 24);
        if ((magic & 0xfffffff0u) == 0x184D2A50u) {          // skippable frame: magic, 4-byte size, payload
            if (n - pos < 8) return false;
            const uint64_t sz = (uint32_t)p[pos + 4] | ((uint32_t)p[pos + 5] << 8) | ((uint32_t)p[pos + 6] << 16) | ((uint64_t)p[pos + 7] << 24);
            if (n - pos - 8 < sz) return false;
            out.push_back({pos, (size_t)(8 + sz), 0, true, true});
            pos += 8 + sz;
            continue;
        }
        if (magic != 0xFD2FB528u) return false;
        size_t q = pos + 4;
        if (q >= n) return false;
        const uint8_t fhd = p[q++];
        if (fhd & 8) return false;
        const bool single = (fhd & 32) != 0, crc = (fhd & 4) != 0;
        if (!single) { if (q >= n) return false; q++; }
        const unsigned did = fhd & 3, didLen = did == 3 ? 4 : did;
        if (n - q < didLen) return false;
        q += didLen;
        unsigned fcsLen = 0;
        if ((fhd >> 6) == 0) fcsLen = single ? 1 : 0; else fcsLen = 1u << (fhd >> 6);
        if (n - q < fcsLen) return false;
        uint64_t fcs = 0;
        for (unsigned k = 0; k < fcsLen; k++) fcs |= (uint64_t)p[q + k] << (8 * k);
        if (fcsLen == 2) fcs += 256;
        q += fcsLen;
        for (;;) {                                          // blocks
            if (n - q < 3) return false;
            const uint32_t bh = (uint32_t)p[q] | ((uint32_t)p[q + 1] << 8) | ((uint32_t)p[q + 2] << 16);
            q += 3;
            const uint32_t bt = (bh >> 1) & 3, bs = bh >> 3;
            if (bt == 3) return false;
            const size_t body = bt == 1 ? 1 : bs;
            if (n - q < body) return false;
            q += body;
            if (bh & 1) break;
        }
        if (crc) { if (n - q < 4) return false; q += 4; }
        out.push_back({pos, q - pos, fcs, fcsLen != 0, false});
        pos = q;
    }
    return true;
}

// Host-buffer batch decode: inputs are packed back to back, copied H2D, decoded, outputs copied back.  A stream whose
// frames all declare their content size (what every encoder here and the reference's EncodeAll write) is cut into its
// frames: every frame gets its own decoder warp and the device output buffer is sized from the declared sizes instead
// of the caller's cap (DecodeAll of a large EncodeAll output is thousands of independent frames, not one serial stream).
int b2c_zstd_decode_chunks(b2c_ctx *ctx, const void *const *srcs, const size_t *src_sizes, void *const *dsts,
                           const size_t *dst_caps, int64_t *sizes_out, size_t n) {
    if (!ctx) return B2C_ERR_NO_DEVICE;
    if (n == 0) return B2C_OK;
    int rc = HostBatch::check(ctx, n, src_sizes, 0xffffffffull);
    if (rc) return rc;
    // work items: one per frame (split inputs) or one per input (everything else)
    struct Item { size_t input; size_t src_off_in_input; uint32_t src_len; uint64_t dst_off_in_input; uint32_t cap; };
    std::vector<Item> items;
    std::vector<size_t> first_item(n + 1, 0);
    std::vector<size_t> out_len(n);
    std::vector<char> split(n, 0);
    std::vector<FrameSpan> fr;
    for (size_t i = 0; i < n; i++) {
        first_item[i] = items.size();
        const uint64_t cap = clamp32(dst_caps[i]);
        fr.clear();
        bool ok = src_sizes[i] > 0 && scan_frames((const uint8_t *)srcs[i], src_sizes[i], fr) && !fr.empty();
        uint64_t total = 0;
        if (ok)
            for (const FrameSpan &f : fr) {
                if (!f.skippable && (!f.has_fcs || f.fcs > 0xffffffffull)) { ok = false; break; }
                total += f.skippable ? 0 : f.fcs;
            }
        if (ok && total > cap) ok = false;               // the serial path reports the reference's "too large" error
        if (ok) {
            split[i] = 1;
            uint64_t o = 0;
            for (const FrameSpan &f : fr) {
                if (f.skippable) continue;
                items.push_back({i, f.off, (uint32_t)f.len, o, (uint32_t)f.fcs});
                o += f.fcs;
            }
            out_len[i] = total;
        } else {
            items.push_back({i, 0, (uint32_t)src_sizes[i], 0, (uint32_t)cap});
            out_len[i] = cap;
        }
    }
    first_item[n] = items.size();
    const size_t m = items.size();
    if (m > 0xffffffffull) return B2C_ERR_ARG;
    HostBatch B(ctx, n, m);
    B.place(src_sizes, 0, out_len.data(), 0);
    for (size_t k = 0; k < m; k++) {
        B.h.src_off[k] = B.in_off[items[k].input] + items[k].src_off_in_input;
        B.h.dst_off[k] = B.out_off[items[k].input] + items[k].dst_off_in_input;
        B.h.src_sizes[k] = items[k].src_len; B.h.dst_caps[k] = items[k].cap;
    }
    if ((rc = B.stage_in(srcs, src_sizes))) return rc;
    ZstdDecParams P = B.params<ZstdDecParams>();
    P.nchunks = (uint32_t)m;
    if ((rc = launch_decode(ctx, P, ctx->stream, B.out_bytes, 0))) return rc;
    std::vector<int64_t> res(m);
    if ((rc = B.results(res.data()))) return rc;
    for (size_t i = 0; i < n; i++) {
        int64_t total = 0;
        for (size_t k = first_item[i]; k < first_item[i + 1]; k++) {
            if (res[k] < 0) {                                                // the first failing frame decides
                // a split frame's capacity is its declared content size: running out of it means the frame is larger
                // than declared, which the reference reports as ErrFrameSizeExceeded (framedec.go:330-412)
                total = (split[i] && res[k] == B2C_ERR_DST_SMALL) ? (int64_t)B2C_ERR_SIZE : res[k];
                break;
            }
            if (split[i] && (uint64_t)res[k] != items[k].cap) { total = B2C_ERR_SIZE; break; }   // declared size not met
            total += res[k];
        }
        sizes_out[i] = total;
    }
    return B.scatter(dsts, sizes_out, dst_caps);
}


// ---- S2 / Snappy blocks ---------------------------------------------------------------------------
size_t b2c_s2_bound(size_t n) {
    // s2.MaxEncodedLen (s2/encode.go:389-418), 64-bit platform; 0 when the block is too large
    if (n > 0xffffffffull) return 0;
    size_t bits = 0;
    for (size_t v = n; v; v >>= 1) bits++;
    size_t r = n + (bits + 7) / 7;
    if (n) r += n < 60 ? 1 : n < (1u << 8) ? 2 : n < (1u << 16) ? 3 : n < (1u << 24) ? 4 : 5;
    return r > 0xffffffffull ? 0 : r;
}

static int launch_s2_encode(b2c_ctx *ctx, int level, int flags, const void *d_src, size_t src_stride,
                            const uint32_t *d_sizes, uint32_t size_all, uint64_t src_total, void *d_dst, size_t dst_stride,
                            int64_t *d_out_sizes, uint32_t nchunks, cudaStream_t st) {
    if (!ctx) return B2C_ERR_NO_DEVICE;
    if (level != B2C_S2_FAST && level != B2C_S2_BETTER && level != B2C_S2_BEST) return B2C_ERR_UNSUPPORTED;
    if (nchunks == 0) return B2C_OK;
    if (dst_stride > 0xffffffffull) return B2C_ERR_ARG;
    CK(cudaSetDevice(ctx->device));
    { int r = ctx_order_begin(ctx, st); if (r) return r; }
    ZstdEncParams P;
    memset(&P, 0, sizeof(P));
    P.src_base = (const uint8_t *)d_src; P.src_stride = src_stride; P.src_sizes = d_sizes; P.src_size_all = size_all;
    P.src_total = src_total;
    P.dst_base = (uint8_t *)d_dst; P.dst_stride = dst_stride; P.dst_cap = (uint32_t)dst_stride;
    P.out_sizes = d_out_sizes; P.nchunks = nchunks; P.blockmax = ENC_MAX_CHUNK;
    P.scratch = ctx->d_scratch.p;
    if (level == B2C_S2_BEST) {     // (its own scratch: four candidate distances per position do not fit the shared set)
        const size_t need = (size_t)ctx->sm_count * LzCfg<LZ_S2BEST>::MIN_CTAS * LzLayout<LZ_S2BEST>::SCRATCH_BYTES;
        { int r = reserve(ctx, ctx->d_s2best, need); if (r) return r; }
        P.scratch = ctx->d_s2best.p;
    }
    { int r = next_counter(ctx, st, &P.counter); if (r) return r; }
    const unsigned sms = (unsigned)ctx->sm_count;
    const bool snappy = (flags & B2C_S2_SNAPPY) != 0;
    if (level == B2C_S2_FAST) {
        const unsigned cap = sms * LzCfg<3>::MIN_CTAS, g1 = cap < nchunks ? cap : nchunks;
        if (snappy) b2c_lz_snappy_fast_kernel<<<g1, LzCfg<3>::NT, LzLayout<3>::SMEM_BYTES, st>>>(P);
        else b2c_lz_s2_fast_kernel<<<g1, LzCfg<3>::NT, LzLayout<3>::SMEM_BYTES, st>>>(P);
    } else if (level == B2C_S2_BETTER) {
        const unsigned cap = sms * LzCfg<4>::MIN_CTAS, g1 = cap < nchunks ? cap : nchunks;
        if (snappy) b2c_lz_snappy_better_kernel<<<g1, LzCfg<4>::NT, LzLayout<4>::SMEM_BYTES, st>>>(P);
        else b2c_lz_s2_better_kernel<<<g1, LzCfg<4>::NT, LzLayout<4>::SMEM_BYTES, st>>>(P);
    } else {
        const unsigned cap = sms * LzCfg<LZ_S2BEST>::MIN_CTAS, g1 = cap < nchunks ? cap : nchunks;
        if (snappy) b2c_lz_snappy_best_kernel<<<g1, LzCfg<LZ_S2BEST>::NT, LzLayout<LZ_S2BEST>::SMEM_BYTES, st>>>(P);
        else b2c_lz_s2_best_kernel<<<g1, LzCfg<LZ_S2BEST>::NT, LzLayout<LZ_S2BEST>::SMEM_BYTES, st>>>(P);
    }
    ctx->launches += 1;
    CK(cudaGetLastError());
    return ctx_order_end(ctx, st);
}

int b2c_s2_encode_device(b2c_ctx *ctx, int level, int flags, const void *d_src, size_t src_stride,
                         const uint32_t *d_sizes, uint32_t size_all, void *d_dst, size_t dst_stride,
                         int64_t *d_out_sizes, uint32_t nchunks, void *stream) {
    return launch_s2_encode(ctx, level, flags, d_src, src_stride, d_sizes, size_all, 0, d_dst, dst_stride, d_out_sizes, nchunks,
                            (cudaStream_t)stream);
}

static int launch_s2_decode(b2c_ctx *ctx, S2DecParams &P, uint64_t span, cudaStream_t st);

// ------------------------------------------------------------------------------------------------ S2 / Snappy streams
// s2.Writer.EncodeBuffer / s2.Reader for whole buffers (s2/writer.go:357-470, s2/reader.go:249-420): the framing format
// around the block codecs -- stream identifier, one chunk per block with the masked CRC32-C of its uncompressed bytes.
size_t b2c_s2_stream_bound(size_t n, size_t block) {
    if (block == 0 || block > 65536) return 0;
    const size_t nb = (n + block - 1) / block;
    return 10 + nb * 8 + nb * (b2c_s2_bound(block) - block) + n;
}

// Device-resident: d_src[0, n) -> a complete stream in d_dst; *d_total (device, 8 bytes) = its length; *d_err (device, 4
// bytes) = 0 or a negative error (B2C_ERR_DST_SMALL).  block <= 65536.  Asynchronous on `stream`.
int b2c_s2_encode_stream_device(b2c_ctx *ctx, int level, int flags, const void *d_src, uint64_t n, uint32_t block, void *d_dst,
                                uint64_t dst_cap, uint64_t *d_total, int32_t *d_err, void *stream) {
    if (!ctx) return B2C_ERR_NO_DEVICE;
    if (level != B2C_S2_FAST && level != B2C_S2_BETTER && level != B2C_S2_BEST) return B2C_ERR_UNSUPPORTED;
    if (block == 0 || block > 65536 || !d_total || !d_err) return B2C_ERR_ARG;
    if (n / block >= 0x7fffffffull || dst_cap < 10) return B2C_ERR_ARG;
    CK(cudaSetDevice(ctx->device));
    cudaStream_t st = (cudaStream_t)stream;
    const uint32_t nblocks = (uint32_t)((n + block - 1) / block);
    const uint32_t sub = nblocks < 4096 ? (nblocks ? nblocks : 1) : 4096u, nsub = (nblocks + sub - 1) / sub;
    const size_t slotB = (b2c_s2_bound(block) + 15) & ~(size_t)15;
    Layout L;
    const size_t oSlots = L.take(slotB * sub), oEnc = L.take(sizeof(int64_t) * sub), oPiece = L.take(sizeof(int64_t) * sub),
                 oCrc = L.take(sizeof(uint32_t) * sub), oScan = L.take(sizeof(uint64_t) * ((size_t)sub + 1)),
                 oBase = L.take(sizeof(uint64_t) * ((size_t)nsub + 1));
    { int r = reserve(ctx, ctx->d_s2s, L.end); if (r) return r; }
    { int r = ctx_order_begin(ctx, st); if (r) return r; }
    uint8_t *B = ctx->d_s2s.p;
    uint64_t *d_base = (uint64_t *)(B + oBase);
    CK(cudaMemsetAsync(d_base, 0, sizeof(uint64_t), st));
    CK(cudaMemsetAsync(d_err, 0, sizeof(int32_t), st));
    const bool snappy = (flags & B2C_S2_SNAPPY) != 0;
    if (nblocks == 0) {      // an empty input: the identifier alone
        const char *magic = snappy ? "\xff\x06\x00\x00sNaPpY" : "\xff\x06\x00\x00S2sTwO";
        CK(cudaMemcpyAsync(d_dst, magic, 10, cudaMemcpyHostToDevice, st));
    }
    for (uint32_t k = 0; k < nsub && nblocks; k++) {
        const uint32_t c0 = k * sub, m = (nblocks - c0 < sub) ? nblocks - c0 : sub;
        const uint8_t *srck = (const uint8_t *)d_src + (uint64_t)c0 * block;
        int r = launch_s2_encode(ctx, level, flags, srck, block, nullptr, block, n - (uint64_t)c0 * block, B + oSlots, slotB,
                                 (int64_t *)(B + oEnc), m, st);
        if (r) return r;
        S2StreamParams P;
        memset(&P, 0, sizeof(P));
        P.src = (const uint8_t *)d_src; P.total = n; P.block = block;
        P.slots = B + oSlots; P.slot_stride = slotB; P.enc_sizes = (const int64_t *)(B + oEnc);
        P.crc = (uint32_t *)(B + oCrc); P.piece = (int64_t *)(B + oPiece); P.offsets = (const uint64_t *)(B + oScan);
        P.base = d_base; P.k = k; P.dst = (uint8_t *)d_dst; P.cap = dst_cap; P.c0 = c0; P.m = m; P.snappy = snappy ? 1u : 0u;
        P.err = d_err;
        b2c_s2_stream_crc_kernel<<<(unsigned)ctx->sm_count * 4, S2S_WARPS * 32, 0, st>>>(P);
        b2c_scan_sizes_kernel<<<1, 1024, 0, st>>>(P.piece, (uint64_t *)(B + oScan), m);
        b2c_s2_stream_place_kernel<<<(unsigned)ctx->sm_count * 8, 256, 0, st>>>(P);
        b2c_frame_base_kernel<<<1, 1, 0, st>>>(d_base, k, (const uint64_t *)(B + oScan), m);
        ctx->launches += 4;
    }
    // total = identifier + all pieces
    b2c_s2_stream_total_kernel<<<1, 1, 0, st>>>(d_base, nsub * (nblocks ? 1u : 0u), d_total);
    CK(cudaGetLastError());
    return ctx_order_end(ctx, st);
}

// Host buffers: src[0, n) -> stream in dst (capacity cap >= b2c_s2_stream_bound); *out_len = stream bytes.  Synchronous.
int b2c_s2_encode_stream(b2c_ctx *ctx, int level, int flags, const void *src, size_t n, uint32_t block, void *dst, size_t cap,
                         size_t *out_len) {
    if (!ctx) return B2C_ERR_NO_DEVICE;
    if (!out_len || block == 0 || block > 65536) return B2C_ERR_ARG;
    CK(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    const size_t bound = b2c_s2_stream_bound(n, block);
    Layout L;
    const size_t oIn = L.take(n), oOut = L.take(bound), oTotal = L.take(sizeof(uint64_t)), oErr = L.take(sizeof(int32_t));
    { int r = reserve(ctx, ctx->d_s2s_io, L.end); if (r) return r; }
    uint8_t *d_in = ctx->d_s2s_io.at<uint8_t>(oIn), *d_out = ctx->d_s2s_io.at<uint8_t>(oOut);
    uint64_t *d_total = ctx->d_s2s_io.at<uint64_t>(oTotal);
    int32_t *d_err = ctx->d_s2s_io.at<int32_t>(oErr);
    if (n) CK(cudaMemcpyAsync(d_in, src, n, cudaMemcpyHostToDevice, st));
    int r = b2c_s2_encode_stream_device(ctx, level, flags, d_in, n, block, d_out, bound, d_total, d_err, st);
    if (r) { cudaStreamSynchronize(st); return r; }
    uint64_t total = 0; int32_t err = 0;
    CK(cudaMemcpyAsync(&total, d_total, sizeof(total), cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(&err, d_err, sizeof(err), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    if (err) return err;
    if (total > cap) return B2C_ERR_DST_SMALL;
    CK(cudaMemcpy(dst, d_out, total, cudaMemcpyDeviceToHost));
    *out_len = (size_t)total;
    return B2C_OK;
}

// Host buffers: a complete S2 / Snappy stream -> its content (s2.Reader over a buffer).  The chunk headers are walked on the
// host (4 bytes each, no data is touched there); the device decodes every block, copies uncompressed chunks and verifies
// all checksums.  Errors are the reader's: B2C_ERR_CORRUPT (ErrCorrupt), B2C_ERR_CRC (ErrCRC), B2C_ERR_UNSUPPORTED
// (reserved unskippable chunk), B2C_ERR_DST_SMALL.
int b2c_s2_decode_stream(b2c_ctx *ctx, const void *src, size_t n, void *dst, size_t cap, size_t *out_len) {
    if (!ctx) return B2C_ERR_NO_DEVICE;
    if (!out_len) return B2C_ERR_ARG;
    const uint8_t *s = (const uint8_t *)src;
    std::vector<S2StreamBlock> blocks;
    uint64_t o = 0, total = 0;
    bool seen = false, snappyFrame = false;
    const uint32_t maxBlock = 4u << 20;                      // s2/s2.go:87 maxBlockSize
    while (o < n) {
        if (o + 4 > n) return B2C_ERR_CORRUPT;               // io.ErrUnexpectedEOF
        const uint32_t typ = s[o], ln = (uint32_t)s[o + 1] | (uint32_t)s[o + 2] << 8 | (uint32_t)s[o + 3] << 16;
        o += 4;
        if (!seen) { if (typ != 0xff) return B2C_ERR_CORRUPT; seen = true; }
        if (typ == 0x00 || typ == 0x01) {
            if (ln < 4 || o + ln > n) return B2C_ERR_CORRUPT;
            S2StreamBlock b;
            b.type = typ; b.crc = (uint32_t)s[o] | (uint32_t)s[o + 1] << 8 | (uint32_t)s[o + 2] << 16 | (uint32_t)s[o + 3] << 24;
            b.src_off = o + 4; b.src_len = ln - 4; b.dst_off = total;
            if (typ == 0x00) {
                uint64_t v = 0; uint32_t k = 0, shift = 0;             // DecodedLen (s2/decode.go:36-49)
                for (;;) {
                    if (k >= b.src_len || k >= 10) return B2C_ERR_CORRUPT;
                    const uint8_t by = s[b.src_off + k++];
                    v |= (uint64_t)(by & 0x7f) << shift;
                    if (by < 0x80) break;
                    shift += 7;
                }
                if (k > 5 || v > 0xffffffffull) return B2C_ERR_CORRUPT;
                if (v > maxBlock || (snappyFrame && v > 65536)) return B2C_ERR_CORRUPT;
                b.dst_len = (uint32_t)v;
            } else {
                if (b.src_len > maxBlock || (snappyFrame && b.src_len > 65536)) return B2C_ERR_CORRUPT;
                b.dst_len = b.src_len;
            }
            total += b.dst_len;
            blocks.push_back(b);
        } else if (typ == 0xff) {
            if (ln != 6 || o + 6 > n) return B2C_ERR_CORRUPT;
            if (memcmp(s + o, "S2sTwO", 6) == 0) snappyFrame = false;
            else if (memcmp(s + o, "sNaPpY", 6) == 0) snappyFrame = true;
            else return B2C_ERR_CORRUPT;
        } else if (typ <= 0x7f) {
            return B2C_ERR_UNSUPPORTED;                        // reserved unskippable chunk (s2/reader.go:386-391)
        } else if (o + ln > n) {
            return B2C_ERR_CORRUPT;                            // skippable chunk / padding cut short
        }
        o += ln;
    }
    if (total > cap) return B2C_ERR_DST_SMALL;
    *out_len = (size_t)total;
    const uint32_t nb = (uint32_t)blocks.size();
    if (nb == 0) return B2C_OK;
    CK(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    Layout L;
    const size_t oIn = L.take(n), oOut = L.take(total + 16), oBlk = L.take(sizeof(S2StreamBlock) * nb),
                 oSrcOff = L.take(8 * (size_t)nb), oDstOff = L.take(8 * (size_t)nb), oSrcSz = L.take(4 * (size_t)nb),
                 oCaps = L.take(4 * (size_t)nb), oRes = L.take(8 * (size_t)nb), oStat = L.take(4 * (size_t)nb);
    { int r = reserve(ctx, ctx->d_s2s_io, L.end); if (r) return r; }
    uint8_t *B = ctx->d_s2s_io.p;
    // compressed blocks go to the block decoder; an uncompressed chunk is handed to it as an empty job (size 0 in, cap 0)
    std::vector<uint64_t> so(nb), dof(nb);
    std::vector<uint32_t> ssz(nb), caps(nb);
    for (uint32_t i = 0; i < nb; i++) {
        so[i] = blocks[i].src_off; dof[i] = blocks[i].dst_off;
        ssz[i] = blocks[i].type == 0 ? blocks[i].src_len : 0; caps[i] = blocks[i].type == 0 ? blocks[i].dst_len : 0;
    }
    CK(cudaMemcpyAsync(B + oIn, src, n, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(B + oBlk, blocks.data(), sizeof(S2StreamBlock) * nb, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(B + oSrcOff, so.data(), 8 * (size_t)nb, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(B + oDstOff, dof.data(), 8 * (size_t)nb, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(B + oSrcSz, ssz.data(), 4 * (size_t)nb, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(B + oCaps, caps.data(), 4 * (size_t)nb, cudaMemcpyHostToDevice, st));
    S2DecParams P;
    memset(&P, 0, sizeof(P));
    P.src_base = B + oIn; P.src_offsets = (const uint64_t *)(B + oSrcOff); P.src_sizes = (const uint32_t *)(B + oSrcSz);
    P.dst_base = B + oOut; P.dst_offsets = (const uint64_t *)(B + oDstOff); P.dst_caps = (const uint32_t *)(B + oCaps);
    P.out_sizes = (int64_t *)(B + oRes); P.nchunks = nb;
    { int r = launch_s2_decode(ctx, P, n, st); if (r) return r; }
    unsigned g2 = (nb + S2S_WARPS - 1) / S2S_WARPS;
    if (g2 > (unsigned)ctx->sm_count * 16) g2 = (unsigned)ctx->sm_count * 16;
    b2c_s2_stream_verify_kernel<<<g2, S2S_WARPS * 32, 0, st>>>((const S2StreamBlock *)(B + oBlk), B + oIn, B + oOut,
                                                                (const int64_t *)(B + oRes), (int32_t *)(B + oStat), nb);
    ctx->launches += 1;
    std::vector<int32_t> stat(nb);
    CK(cudaMemcpyAsync(stat.data(), B + oStat, 4 * (size_t)nb, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    for (uint32_t i = 0; i < nb; i++)
        if (stat[i]) return stat[i] == -4 ? B2C_ERR_CORRUPT : stat[i];      // (a block longer than its declared length is corrupt)
    CK(cudaMemcpy(dst, B + oOut, total, cudaMemcpyDeviceToHost));
    return B2C_OK;
}

// S2 block decode launch.  span = bytes of the input layout (blocks lie inside [0, span) at increasing, non-overlapping offsets) or
// 0 when the host does not know it.  With a span the staged form runs first (tag walk one lane per block, execution one warp per
// block); the one-warp kernel then takes what they left (large or unusual blocks, errors).
static int launch_s2_decode(b2c_ctx *ctx, S2DecParams &P, uint64_t span, cudaStream_t st) {
    const uint32_t n = P.nchunks;
    // (a call with per-block source offsets passes span 0: the element records are placed by the offsets, whose extent the
    // host does not know, so such a call runs the one-warp kernel alone)
    const bool staged = ctx->dec_staged && span > 0 && span <= ((uint64_t)8 << 30);
    ctx->s2d_last = staged;
    if (staged) {
        Layout L;
        const size_t recBytes = ((size_t)(span / 3) + n + 16) * sizeof(uint64_t);
        const size_t oHead = L.take((size_t)n * sizeof(S2Head)), oRec = L.take(recBytes);
        { int r = ctx_order_begin(ctx, st); if (r) return r; }
        int rc = reserve(ctx, ctx->d_s2d, oRec + recBytes);
        if (rc) return rc;
        P.heads = ctx->d_s2d.at<S2Head>(oHead);
        P.recs = ctx->d_s2d.at<uint64_t>(oRec);
        b2c_s2_walk_kernel<<<(n + 31) / 32, 32, 0, st>>>(P);
        b2c_s2_exec_kernel<<<(n + S2DEC_WARPS - 1) / S2DEC_WARPS, S2DEC_WARPS * 32, 0, st>>>(P);
        ctx->launches += 2;
    }
    unsigned grid = (n + S2DEC_WARPS - 1) / S2DEC_WARPS, maxGrid = (unsigned)ctx->sm_count * 16;
    if (grid > maxGrid) grid = maxGrid;
    b2c_s2_decode_kernel<<<grid, S2DEC_WARPS * 32, 0, st>>>(P);
    ctx->launches += 1;
    CK(cudaGetLastError());
    if (staged) return ctx_order_end(ctx, st);
    return B2C_OK;
}

int b2c_s2_decode_device(b2c_ctx *ctx, const void *d_src, size_t src_stride, const uint64_t *d_src_offsets,
                         const uint32_t *d_src_sizes, void *d_dst, size_t dst_stride, const uint64_t *d_dst_offsets,
                         uint32_t dst_cap, int64_t *d_out_sizes, uint32_t nchunks, void *stream) {
    if (!ctx) return B2C_ERR_NO_DEVICE;
    if (!d_src_sizes || !d_out_sizes) return B2C_ERR_ARG;
    if (nchunks == 0) return B2C_OK;
    CK(cudaSetDevice(ctx->device));
    S2DecParams P;
    memset(&P, 0, sizeof(P));
    P.src_base = (const uint8_t *)d_src; P.src_stride = src_stride; P.src_offsets = d_src_offsets; P.src_sizes = d_src_sizes;
    P.dst_base = (uint8_t *)d_dst; P.dst_stride = dst_stride; P.dst_offsets = d_dst_offsets; P.dst_cap = dst_cap;
    P.out_sizes = d_out_sizes; P.nchunks = nchunks;
    return launch_s2_decode(ctx, P, d_src_offsets ? 0 : (uint64_t)nchunks * src_stride, (cudaStream_t)stream);
}

// Host-buffer batches for the block API (s2.Encode / s2.EncodeSnappy / s2.Decode per element).  Inputs are packed
// back to back on the device, outputs land in per-element slots; one kernel per call.
static int s2_host_batch(b2c_ctx *ctx, bool encode, int level, int flags, const void *const *srcs, const size_t *src_sizes,
                         void *const *dsts, const size_t *dst_caps, int64_t *sizes_out, size_t n) {
    if (!ctx) return B2C_ERR_NO_DEVICE;
    if (n == 0) return B2C_OK;
    int rc = HostBatch::check(ctx, n, src_sizes, 0xffffffffull);
    if (rc) return rc;
    HostBatch B(ctx, n, n);
    // encode: fixed strides (the kernel addresses chunks by stride)
    B.place_items(src_sizes, encode ? ENC_MAX_CHUNK : 0, dst_caps, encode ? kSlot : 0);
    std::vector<size_t> lens(src_sizes, src_sizes + n);
    for (size_t i = 0; i < n; i++)
        if (encode && src_sizes[i] > ENC_MAX_CHUNK) { B.h.src_sizes[i] = ENC_MAX_CHUNK + 1; lens[i] = 0; }   // reported as too big
    if ((rc = B.stage_in(srcs, lens.data()))) return rc;
    if (encode)
        rc = b2c_s2_encode_device(ctx, level, flags, ctx->d_dec_in.p, ENC_MAX_CHUNK, B.d.src_sizes, 0, ctx->d_dec_out.p, kSlot,
                                  B.d.res, (uint32_t)n, ctx->stream);
    else {
        S2DecParams P = B.params<S2DecParams>();
        P.nchunks = (uint32_t)n;
        rc = launch_s2_decode(ctx, P, B.in_bytes, ctx->stream);
    }
    if (rc || (rc = B.results(sizes_out))) return rc;
    return B.scatter(dsts, sizes_out, dst_caps);
}

int b2c_s2_encode_chunks(b2c_ctx *ctx, int level, int flags, const void *const *srcs, const size_t *src_sizes,
                         void *const *dsts, const size_t *dst_caps, int64_t *sizes_out, size_t n) {
    if (level != B2C_S2_FAST && level != B2C_S2_BETTER && level != B2C_S2_BEST) return ctx ? B2C_ERR_UNSUPPORTED : B2C_ERR_NO_DEVICE;
    return s2_host_batch(ctx, true, level, flags, srcs, src_sizes, dsts, dst_caps, sizes_out, n);
}
int b2c_s2_decode_chunks(b2c_ctx *ctx, const void *const *srcs, const size_t *src_sizes, void *const *dsts,
                         const size_t *dst_caps, int64_t *sizes_out, size_t n) {
    return s2_host_batch(ctx, false, 0, 0, srcs, src_sizes, dsts, dst_caps, sizes_out, n);
}


// ---- LZ4 / LZ4s -> S2 / Snappy block conversion ---------------------------------------------------------
// Passes of next_pass(); rec_base (device) holds every block's first record when the host knows the sizes, otherwise every
// block gets room for a block of max_src bytes.
static int launch_lz4_convert(b2c_ctx *ctx, LzcParams P, uint32_t n, uint64_t max_src, const uint64_t *h_rec_base,
                              cudaStream_t st) {
    const uint64_t per = (P.lz4s ? max_src / 2 : max_src / 3) + 1;
    { int r = ctx_order_begin(ctx, st); if (r) return r; }
    for (uint32_t c0 = 0, c1; c0 < n; c0 = c1) {
        const uint64_t recs = next_pass(c0, n, h_rec_base, per, sizeof(LzcRec), &c1);
        const uint32_t m = c1 - c0;
        Layout L;
        const size_t oHead = L.take((size_t)m * sizeof(LzcHead)), oRec = L.take((size_t)recs * sizeof(LzcRec));
        { int r = reserve(ctx, ctx->d_lzc, L.end); if (r) return r; }
        P.c0 = c0; P.nchunks = m; P.rec_per = per;
        P.heads = ctx->d_lzc.at<LzcHead>(oHead);
        P.recs = ctx->d_lzc.at<LzcRec>(oRec);
        b2c_lz4_cvt_walk_kernel<<<(m + 31) / 32, 32, 0, st>>>(P);
        b2c_lz4_cvt_emit_kernel<<<(m + LZC_EMIT_WARPS - 1) / LZC_EMIT_WARPS, LZC_EMIT_WARPS * 32, 0, st>>>(P);
        ctx->launches += 2;
        CK(cudaGetLastError());
    }
    return ctx_order_end(ctx, st);
}

int b2c_s2_convert_lz4_device(b2c_ctx *ctx, int format, int flags, const void *d_src, size_t src_stride,
                              const uint64_t *d_src_offsets, const uint32_t *d_src_sizes, void *d_dst, size_t dst_stride,
                              const uint64_t *d_dst_offsets, uint32_t dst_cap, int64_t *d_out_sizes, int64_t *d_decoded,
                              uint32_t nchunks, void *stream) {
    if (!ctx) return B2C_ERR_NO_DEVICE;
    if ((format != B2C_LZ4 && format != B2C_LZ4S) || (flags & ~B2C_S2_SNAPPY)) return B2C_ERR_ARG;
    if (!d_src_sizes || !d_out_sizes || !d_decoded || src_stride == 0 || src_stride > 0xffffffffull) return B2C_ERR_ARG;
    if (nchunks == 0) return B2C_OK;
    CK(cudaSetDevice(ctx->device));
    LzcParams P;
    memset(&P, 0, sizeof(P));
    P.src_base = (const uint8_t *)d_src; P.src_stride = src_stride; P.src_offsets = d_src_offsets; P.src_sizes = d_src_sizes;
    P.dst_base = (uint8_t *)d_dst; P.dst_stride = dst_stride; P.dst_offsets = d_dst_offsets; P.dst_cap = dst_cap;
    P.out_sizes = d_out_sizes; P.decoded = d_decoded;
    P.lz4s = format == B2C_LZ4S; P.snappy = (flags & B2C_S2_SNAPPY) != 0;
    return launch_lz4_convert(ctx, P, nchunks, src_stride, nullptr, (cudaStream_t)stream);
}

int b2c_s2_convert_lz4_chunks(b2c_ctx *ctx, int format, int flags, const void *const *srcs, const size_t *src_sizes,
                              void *const *dsts, const size_t *dst_caps, int64_t *sizes_out, int64_t *decoded_out, size_t n) {
    if (!ctx) return B2C_ERR_NO_DEVICE;
    if ((format != B2C_LZ4 && format != B2C_LZ4S) || (flags & ~B2C_S2_SNAPPY)) return B2C_ERR_ARG;
    if (n == 0) return B2C_OK;
    int rc = HostBatch::check(ctx, n, src_sizes, 0xffffffffull);
    if (rc) return rc;
    const bool lz4s = format == B2C_LZ4S;
    HostBatch B(ctx, n, n, {(n + 1) * sizeof(uint64_t)});            // + the record bases
    const size_t oDec = B.L.take(n * sizeof(int64_t));               // decoded lengths (device only)
    B.place_items(src_sizes, 0, dst_caps, 0);
    uint64_t *rec_base = B.h_at<uint64_t>(B.ex[0]);
    rec_base[0] = 0;
    for (size_t i = 0; i < n; i++) rec_base[i + 1] = rec_base[i] + (lz4s ? src_sizes[i] / 2 : src_sizes[i] / 3) + 1;
    if ((rc = B.stage_in(srcs, src_sizes))) return rc;
    LzcParams P = B.params<LzcParams>();
    P.decoded = B.d_at<int64_t>(oDec);
    P.rec_base = B.d_at<uint64_t>(B.ex[0]);
    P.lz4s = lz4s; P.snappy = (flags & B2C_S2_SNAPPY) != 0;
    if ((rc = launch_lz4_convert(ctx, P, (uint32_t)n, 0, rec_base, ctx->stream))) return rc;
    CK(cudaMemcpyAsync(decoded_out, P.decoded, n * sizeof(int64_t), cudaMemcpyDeviceToHost, ctx->stream));
    if ((rc = B.results(sizes_out))) return rc;
    return B.scatter(dsts, sizes_out, dst_caps);
}

// ---- inflate: raw DEFLATE / zlib / gzip -------------------------------------------------------------------------
// Passes of next_pass(); rec_base (device) holds every input's first record when the host knows the sizes, otherwise every
// input gets room for max_src bytes into cap.
static int launch_inflate(b2c_ctx *ctx, InfParams P, uint32_t n, uint64_t max_src, uint64_t cap, const uint64_t *h_rec_base,
                          cudaStream_t st) {
    const uint64_t per = inf_rec_cap(max_src, cap);
    { int r = ctx_order_begin(ctx, st); if (r) return r; }
    for (uint32_t c0 = 0, c1; c0 < n; c0 = c1) {
        const uint64_t recs = next_pass(c0, n, h_rec_base, per, sizeof(InfRec), &c1);
        const uint32_t m = c1 - c0;
        Layout L;
        const size_t oHead = L.take((size_t)m * sizeof(InfHead)), oRec = L.take((size_t)recs * sizeof(InfRec));
        { int r = reserve(ctx, ctx->d_inf, L.end); if (r) return r; }
        P.c0 = c0; P.nchunks = m; P.rec_per = per;
        P.heads = ctx->d_inf.at<InfHead>(oHead);
        P.recs = ctx->d_inf.at<InfRec>(oRec);
        b2c_inflate_walk_kernel<<<(m + INF_WALK_LANES - 1) / INF_WALK_LANES, INF_WALK_LANES, 0, st>>>(P);
        b2c_inflate_exec_kernel<<<(m + INF_WARPS - 1) / INF_WARPS, INF_WARPS * 32, 0, st>>>(P);
        b2c_inflate_check_kernel<<<(m + INF_WARPS - 1) / INF_WARPS, INF_WARPS * 32, 0, st>>>(P);
        ctx->launches += 3;
        CK(cudaGetLastError());
    }
    return ctx_order_end(ctx, st);
}
static bool flate_args_ok(int format, int flags) {
    return (format == B2C_FLATE_RAW || format == B2C_FLATE_ZLIB || format == B2C_FLATE_GZIP) && !(flags & ~B2C_GZIP_SINGLE);
}

int b2c_flate_decode_device(b2c_ctx *ctx, int format, int flags, const void *d_src, size_t src_stride,
                            const uint64_t *d_src_offsets, const uint32_t *d_src_sizes, void *d_dst, size_t dst_stride,
                            const uint64_t *d_dst_offsets, uint32_t dst_cap, int64_t *d_out_sizes, uint32_t nchunks, void *stream) {
    if (!ctx) return B2C_ERR_NO_DEVICE;
    if (!flate_args_ok(format, flags)) return B2C_ERR_ARG;
    if (!d_src_sizes || !d_out_sizes || src_stride == 0 || src_stride > 0xffffffffull) return B2C_ERR_ARG;
    if (nchunks == 0) return B2C_OK;
    CK(cudaSetDevice(ctx->device));
    InfParams P;
    memset(&P, 0, sizeof(P));
    P.src_base = (const uint8_t *)d_src; P.src_stride = src_stride; P.src_offsets = d_src_offsets; P.src_sizes = d_src_sizes;
    P.dst_base = (uint8_t *)d_dst; P.dst_stride = dst_stride; P.dst_offsets = d_dst_offsets; P.dst_cap = dst_cap;
    P.out_sizes = d_out_sizes;
    P.format = format; P.multistream = !(flags & B2C_GZIP_SINGLE);
    return launch_inflate(ctx, P, nchunks, src_stride, dst_cap, nullptr, (cudaStream_t)stream);
}

int b2c_flate_decode_chunks(b2c_ctx *ctx, int format, int flags, const void *const *srcs, const size_t *src_sizes,
                            void *const *dsts, const size_t *dst_caps, int64_t *sizes_out, size_t n) {
    if (!ctx) return B2C_ERR_NO_DEVICE;
    if (!flate_args_ok(format, flags)) return B2C_ERR_ARG;
    if (n == 0) return B2C_OK;
    int rc = HostBatch::check(ctx, n, src_sizes, 0xffffffffull);
    if (rc) return rc;
    HostBatch B(ctx, n, n, {(n + 1) * sizeof(uint64_t)});            // + the record bases
    B.place_items(src_sizes, 0, dst_caps, 0);
    uint64_t *rec_base = B.h_at<uint64_t>(B.ex[0]);
    rec_base[0] = 0;
    for (size_t i = 0; i < n; i++) rec_base[i + 1] = rec_base[i] + inf_rec_cap(src_sizes[i], B.h.dst_caps[i]);
    if ((rc = B.stage_in(srcs, src_sizes))) return rc;
    InfParams P = B.params<InfParams>();
    P.rec_base = B.d_at<uint64_t>(B.ex[0]);
    P.format = format; P.multistream = !(flags & B2C_GZIP_SINGLE);
    if ((rc = launch_inflate(ctx, P, (uint32_t)n, 0, 0, rec_base, ctx->stream))) return rc;
    if ((rc = B.results(sizes_out))) return rc;
    return B.scatter(dsts, sizes_out, dst_caps);
}

// ---- stateless deflate: flate.StatelessDeflate / gzip at StatelessCompression ---------------------------------------
// Block slot g = input * max_blocks + k; one pass parses and encodes the slots [g0, g1), at most kDflPassSlots of them
// (about 1 GiB of tokens).  Each input's bit writer lives in d_dfl, so an input whose blocks span passes continues.
static const uint64_t kDflPassSlots = 8192;
size_t b2c_flate_stateless_bound(size_t n, size_t dict_len) {
    (void)dict_len;                                     // a dict only moves the first cut: at most one block more
    return n + 8 * (n / DFL_STEP + 3) + 16;
}
static int launch_deflate(b2c_ctx *ctx, DflParams P, uint32_t n, const void *hdr, size_t hlen, cudaStream_t st) {
    Layout L;
    const size_t oState = L.take((size_t)n * sizeof(DflState)), oHdr = L.take(hlen ? hlen : 1);
    const uint64_t total = (uint64_t)n * P.max_blocks;
    const uint64_t per = total < kDflPassSlots ? total : kDflPassSlots;
    const size_t oSlots = L.take((size_t)per * sizeof(DflSlot)), oTok = L.take((size_t)per * DFL_SLOT_TOKENS * 4);
    { int r = reserve(ctx, ctx->d_dfl, L.end); if (r) return r; }
    { int r = ctx_order_begin(ctx, st); if (r) return r; }
    P.state = ctx->d_dfl.at<DflState>(oState);
    P.slots = ctx->d_dfl.at<DflSlot>(oSlots);
    P.tokens = ctx->d_dfl.at<uint32_t>(oTok);
    P.hdr = ctx->d_dfl.p + oHdr; P.hlen = (uint32_t)hlen;
    if (hlen) CK(cudaMemcpyAsync(ctx->d_dfl.p + oHdr, hdr, hlen, cudaMemcpyHostToDevice, st));
    for (uint64_t g0 = 0; g0 < total; g0 += per) {
        P.g0 = g0; P.g1 = g0 + per < total ? g0 + per : total;
        const uint32_t i0 = (uint32_t)(P.g0 / P.max_blocks), i1 = (uint32_t)((P.g1 + P.max_blocks - 1) / P.max_blocks);
        b2c_deflate_parse_kernel<<<(unsigned)((P.g1 - P.g0 + DFL_PARSE_WARPS - 1) / DFL_PARSE_WARPS), DFL_PARSE_WARPS * 32, 0, st>>>(P, n);
        b2c_deflate_encode_kernel<<<(i1 - i0 + DFL_ENCODE_LANES - 1) / DFL_ENCODE_LANES, DFL_ENCODE_LANES, 0, st>>>(P, i0, i1);
        ctx->launches += 2;
        CK(cudaGetLastError());
    }
    b2c_deflate_crc_kernel<<<(n + DFL_CRC_WARPS - 1) / DFL_CRC_WARPS, DFL_CRC_WARPS * 32, 0, st>>>(P, n);
    ctx->launches += 1;
    CK(cudaGetLastError());
    return ctx_order_end(ctx, st);
}
static bool deflate_args_ok(int format, int flags, const void *hdr, size_t hlen) {
    if (flags != 0 || (format != B2C_FLATE_RAW && format != B2C_FLATE_GZIP)) return false;
    if (format == B2C_FLATE_GZIP) return hdr && hlen >= 10 && hlen < (1u << 20);
    return hlen == 0;
}

int b2c_flate_stateless_device(b2c_ctx *ctx, int format, int flags, const void *d_src, size_t src_stride,
                               const uint64_t *d_src_offsets, const uint32_t *d_src_sizes, const uint8_t *d_eof,
                               const void *d_dict, const uint64_t *d_dict_offsets, const uint32_t *d_dict_sizes,
                               const void *hdr, size_t hlen, void *d_dst, size_t dst_stride, const uint64_t *d_dst_offsets,
                               uint32_t dst_cap, int64_t *d_out_sizes, const uint32_t *d_crc_in, uint32_t *d_crc_out,
                               uint32_t nchunks, void *stream) {
    if (!ctx) return B2C_ERR_NO_DEVICE;
    if (!deflate_args_ok(format, flags, hdr, hlen)) return B2C_ERR_ARG;
    if (!d_src_sizes || !d_out_sizes || src_stride == 0 || src_stride > 0xffffffffull) return B2C_ERR_ARG;
    if (d_dict_sizes && (!d_dict || !d_dict_offsets)) return B2C_ERR_ARG;
    if (format == B2C_FLATE_GZIP && (d_dict_sizes || d_eof)) return B2C_ERR_ARG;       // a gzip member has neither
    if (nchunks == 0) return B2C_OK;
    CK(cudaSetDevice(ctx->device));
    DflParams P;
    memset(&P, 0, sizeof(P));
    P.src_base = (const uint8_t *)d_src; P.src_stride = src_stride; P.src_offsets = d_src_offsets; P.src_sizes = d_src_sizes;
    P.dict_base = (const uint8_t *)d_dict; P.dict_offsets = d_dict_offsets; P.dict_sizes = d_dict_sizes;
    P.eof = d_eof;
    P.dst_base = (uint8_t *)d_dst; P.dst_stride = dst_stride; P.dst_offsets = d_dst_offsets; P.dst_cap = dst_cap;
    P.out_sizes = d_out_sizes; P.crc_in = d_crc_in; P.crc_out = d_crc_out;
    P.format = format;
    const uint32_t mb = dfl_blocks(src_stride, d_dict_sizes ? DFL_DICT : 0);
    P.max_blocks = mb ? mb : 1;
    return launch_deflate(ctx, P, nchunks, hdr, hlen, (cudaStream_t)stream);
}

int b2c_flate_stateless_chunks(b2c_ctx *ctx, int format, int flags, const void *const *srcs, const size_t *src_sizes,
                               const uint8_t *eof, const void *const *dicts, const size_t *dict_sizes, const void *hdr,
                               size_t hlen, void *const *dsts, const size_t *dst_caps, int64_t *sizes_out,
                               const uint32_t *crc_in, uint32_t *crc_out, size_t n) {
    if (!ctx) return B2C_ERR_NO_DEVICE;
    if (!deflate_args_ok(format, flags, hdr, hlen)) return B2C_ERR_ARG;
    if (n == 0) return B2C_OK;
    if (n > 0xffffffffull || (dicts != nullptr) != (dict_sizes != nullptr)) return B2C_ERR_ARG;
    if (format == B2C_FLATE_GZIP && (dicts || eof)) return B2C_ERR_ARG;      // a gzip member has neither
    int rc = HostBatch::check(ctx, n, src_sizes, 0xffffffffull);
    if (rc) return rc;
    // + dict offsets | dict sizes | eof flags | CRC-32 seeds | CRC-32 results; the dict tails follow, gathered on their own
    HostBatch B(ctx, n, n, {n * 8, n * 4, n, n * 4, n * 4});
    B.place_items(src_sizes, 0, dst_caps, 0);
    uint64_t *dict_off = B.h_at<uint64_t>(B.ex[0]);
    uint32_t *dict_sz = B.h_at<uint32_t>(B.ex[1]);
    uint8_t *h_eof = B.h_at<uint8_t>(B.ex[2]);
    uint64_t db = 0;
    uint32_t mb = 1;
    std::vector<const void *> dp(n);
    std::vector<size_t> dl(n);
    for (size_t i = 0; i < n; i++) {
        dl[i] = dicts ? (dict_sizes[i] > DFL_DICT ? DFL_DICT : dict_sizes[i]) : 0;   // only the last 8 KiB count
        dp[i] = dl[i] ? (const uint8_t *)dicts[i] + (dict_sizes[i] - dl[i]) : nullptr;
        dict_off[i] = db; dict_sz[i] = (uint32_t)dl[i];
        const uint32_t b = dfl_blocks(src_sizes[i], (uint32_t)dl[i]);
        if (b > mb) mb = b;
        db += (dl[i] + 15) & ~(size_t)15;
        h_eof[i] = eof ? eof[i] : 1;
    }
    if (crc_in) memcpy(B.h_at<uint32_t>(B.ex[3]), crc_in, n * 4);
    const size_t oDict = B.L.take(db + 16);
    if ((rc = B.stage_in(srcs, src_sizes))) return rc;
    if (dicts && (rc = gather_h2d(ctx, dp.data(), dl.data(), dict_off, n, B.d_at<uint8_t>(oDict), (size_t)db, ctx->stream))) return rc;
    DflParams P = B.params<DflParams>();
    if (dicts) {
        P.dict_base = B.d_at<uint8_t>(oDict); P.dict_offsets = B.d_at<uint64_t>(B.ex[0]);
        P.dict_sizes = B.d_at<uint32_t>(B.ex[1]);
    }
    P.eof = B.d_at<uint8_t>(B.ex[2]);
    P.crc_in = crc_in ? B.d_at<uint32_t>(B.ex[3]) : nullptr;
    P.crc_out = B.d_at<uint32_t>(B.ex[4]);
    P.format = format; P.max_blocks = mb;
    if ((rc = launch_deflate(ctx, P, (uint32_t)n, hdr, hlen, ctx->stream))) return rc;
    if (crc_out) CK(cudaMemcpyAsync(crc_out, P.crc_out, n * 4, cudaMemcpyDeviceToHost, ctx->stream));
    if ((rc = B.results(sizes_out))) return rc;
    return B.scatter(dsts, sizes_out, dst_caps);
}

// ---- BestSpeed: flate.NewWriter(w, 1), zlib / gzip.NewWriterLevel(w, BestSpeed) ------------------------------------
// One lane per input.  Its scratch -- a 2^15-entry int32 table, a window's tokens, a DflSlot and a DflState, about 385 KiB
// -- is in d_dfl; a batch whose lanes need more than kDflL1PassBytes runs in passes over its inputs, each pass's tables
// zeroed before it.
static const uint64_t kDflL1PassBytes = (uint64_t)4 << 30;
static const size_t kDflL1LaneBytes = DFL_L1_TABLE * 4 + DFL_L1_TOKENS * 4 + sizeof(DflSlot) + sizeof(DflState);
// The bound.  storeFast writes each window as one block, and no block is more than 176 bytes longer than the window:
//  - stored: 4 bytes of LEN / NLEN, the 3-bit header and its byte padding, and up to 15 bits of the EOB the block before
//    owed: len + 8.
//  - dynamic: chosen only when its exact size (reuseSize or the new table's header and codes, or the fixed size) is below
//    the stored size, (len + 5) * 8 bits; with the owed EOB, len + 8.
//  - Huffman-only: chosen on an estimate, estBits < (len + 5) * 8, where estBits counts the window's codes and the EOB at
//    their real lengths plus either the table in force's real header (reuse) or a guessed 560-bit header.  A new header
//    for 257 literal and 1 offset code lengths has 17 + 19 * 3 bits and at most 7 bits per code length (repeat codes
//    carry fewer per length), 1 880 bits, so the block is at most 1 320 bits over its estimate: with the owed EOB,
//    len + 5 + 168 < len + 176.
// Close adds the final empty block, its owed EOB and the last partial byte: 4 bytes.  zlib adds 6 bytes, gzip hlen + 8.
size_t b2c_flate_best_speed_bound(size_t n) { return n + 176 * (n / DFL_L1_WINDOW + 1) + 4; }

static int launch_best_speed(b2c_ctx *ctx, DflParams P, uint32_t n, const void *hdr, size_t hlen, cudaStream_t st) {
    const uint32_t maxLanes = (uint32_t)(kDflL1PassBytes / kDflL1LaneBytes), passes = (n + maxLanes - 1) / maxLanes,
                   lanes = (n + passes - 1) / passes;
    Layout L;
    const size_t oTab = L.take((size_t)lanes * DFL_L1_TABLE * 4), oTok = L.take((size_t)lanes * DFL_L1_TOKENS * 4),
                 oSlots = L.take((size_t)lanes * sizeof(DflSlot)), oState = L.take((size_t)lanes * sizeof(DflState)),
                 oHdr = L.take(hlen ? hlen : 1);
    { int r = reserve(ctx, ctx->d_dfl, L.end); if (r) return r; }
    { int r = ctx_order_begin(ctx, st); if (r) return r; }
    int32_t *tables = ctx->d_dfl.at<int32_t>(oTab);
    P.tokens = ctx->d_dfl.at<uint32_t>(oTok);
    P.slots = ctx->d_dfl.at<DflSlot>(oSlots);
    P.state = ctx->d_dfl.at<DflState>(oState);
    P.hdr = ctx->d_dfl.p + oHdr; P.hlen = (uint32_t)hlen;
    if (hlen) CK(cudaMemcpyAsync(ctx->d_dfl.p + oHdr, hdr, hlen, cudaMemcpyHostToDevice, st));
    for (uint32_t i0 = 0; i0 < n; i0 += lanes) {
        const uint32_t i1 = n - i0 < lanes ? n : i0 + lanes;
        CK(cudaMemsetAsync(tables, 0, (size_t)(i1 - i0) * DFL_L1_TABLE * 4, st));
        b2c_deflate_l1_kernel<<<(i1 - i0 + DFL_ENCODE_LANES - 1) / DFL_ENCODE_LANES, DFL_ENCODE_LANES, 0, st>>>(P, tables, i0, i1);
        ctx->launches += 1;
        CK(cudaGetLastError());
    }
    b2c_deflate_l1_check_kernel<<<(n + DFL_CRC_WARPS - 1) / DFL_CRC_WARPS, DFL_CRC_WARPS * 32, 0, st>>>(P, n);
    ctx->launches += 1;
    CK(cudaGetLastError());
    return ctx_order_end(ctx, st);
}
static bool best_speed_args_ok(int format, int flags, const void *hdr, size_t hlen) {
    if (flags != 0 || (format != B2C_FLATE_RAW && format != B2C_FLATE_ZLIB && format != B2C_FLATE_GZIP)) return false;
    if (format == B2C_FLATE_GZIP) return hdr && hlen >= 10 && hlen < (1u << 20);
    return hlen == 0;
}

int b2c_flate_best_speed_device(b2c_ctx *ctx, int format, int flags, const void *d_src, size_t src_stride,
                                const uint64_t *d_src_offsets, const uint32_t *d_src_sizes, const void *hdr, size_t hlen,
                                void *d_dst, size_t dst_stride, const uint64_t *d_dst_offsets, uint32_t dst_cap,
                                int64_t *d_out_sizes, uint32_t *d_check_out, uint32_t nchunks, void *stream) {
    if (!ctx) return B2C_ERR_NO_DEVICE;
    if (!best_speed_args_ok(format, flags, hdr, hlen)) return B2C_ERR_ARG;
    if (!d_src_sizes || !d_out_sizes || src_stride == 0 || src_stride > 0xffffffffull) return B2C_ERR_ARG;
    if (nchunks == 0) return B2C_OK;
    CK(cudaSetDevice(ctx->device));
    DflParams P;
    memset(&P, 0, sizeof(P));
    P.src_base = (const uint8_t *)d_src; P.src_stride = src_stride; P.src_offsets = d_src_offsets; P.src_sizes = d_src_sizes;
    P.dst_base = (uint8_t *)d_dst; P.dst_stride = dst_stride; P.dst_offsets = d_dst_offsets; P.dst_cap = dst_cap;
    P.out_sizes = d_out_sizes; P.crc_out = d_check_out;
    P.format = format;
    return launch_best_speed(ctx, P, nchunks, hdr, hlen, (cudaStream_t)stream);
}

int b2c_flate_best_speed_chunks(b2c_ctx *ctx, int format, int flags, const void *const *srcs, const size_t *src_sizes,
                                const void *hdr, size_t hlen, void *const *dsts, const size_t *dst_caps, int64_t *sizes_out,
                                uint32_t *check_out, size_t n) {
    if (!ctx) return B2C_ERR_NO_DEVICE;
    if (!best_speed_args_ok(format, flags, hdr, hlen)) return B2C_ERR_ARG;
    if (n == 0) return B2C_OK;
    int rc = HostBatch::check(ctx, n, src_sizes, 0xffffffffull);
    if (rc) return rc;
    // an input over the cap is not staged: the lane refuses it from its size alone
    std::vector<size_t> staged(src_sizes, src_sizes + n);
    for (size_t i = 0; i < n; i++) if (staged[i] > DFL_L1_MAX_INPUT) staged[i] = 0;
    HostBatch B(ctx, n, n, {n * 4});                                  // + the checksums
    B.place_items(staged.data(), 0, dst_caps, 0);
    for (size_t i = 0; i < n; i++) B.h.src_sizes[i] = (uint32_t)src_sizes[i];
    if ((rc = B.stage_in(srcs, staged.data()))) return rc;
    DflParams P = B.params<DflParams>();
    P.crc_out = B.d_at<uint32_t>(B.ex[0]);
    P.format = format;
    if ((rc = launch_best_speed(ctx, P, (uint32_t)n, hdr, hlen, ctx->stream))) return rc;
    if (check_out) CK(cudaMemcpyAsync(check_out, P.crc_out, n * 4, cudaMemcpyDeviceToHost, ctx->stream));
    if ((rc = B.results(sizes_out))) return rc;
    return B.scatter(dsts, sizes_out, dst_caps);
}

// ---- HuffmanOnly / NoCompression: flate.NewWriter(w, -2 | 0), zlib / gzip.NewWriterLevel(w, -2 | 0) -----------------
// Window slot = input * max_windows + k (max_windows from src_stride, or from the largest input of a _chunks call), one
// DflNolzWin record each in d_dfl; a batch whose records need more than kDflNolzPassBytes runs in passes over whole
// inputs (an input of under 4 GiB has at most 131 072 windows, 230 MiB of records).
static const uint64_t kDflNolzPassBytes = (uint64_t)4 << 30;
// The bound.  Every window is one block.
//  - Level 0: stored blocks, len + 5 bytes each, then Close's 03 00.
//  - Level -2, stored: up to 15 bits of the EOB the block before owed, the 3-bit header and its byte's end, LEN / NLEN:
//    len + 7 bytes.
//  - Level -2, Huffman: chosen only when estBits, which counts the window's codes under its own table (EOB included) or
//    the reused table's codes, is below the stored size (len + 5) * 8.  A reused table adds its EOB and the owed EOB: 30
//    bits.  A new table adds the owed EOB and a real header of at most 17 + 19 * 3 + 258 * 7 = 1 880 bits; estBits guessed
//    560 bits for it when no table was in force, but only lastHeader -- a header that can be much shorter -- when it
//    replaces one, so the block can exceed the stored size by up to 1 894 bits, not only 1 320: len + 242 bytes.
// Close adds 10 bits and the last partial byte: 2 bytes.  zlib adds 6 bytes, gzip hlen + 8.
size_t b2c_flate_nolz_bound(int level, size_t n) {
    if (level == 0) return n + 5 * (n / DFL_NOLZ_WINDOW_STORE + 1) + 2;
    if (level == -2) return n + 242 * (n / DFL_NOLZ_WINDOW_HUFF + 1) + 2;
    return 0;
}

static int launch_nolz(b2c_ctx *ctx, DflNolzParams P, uint32_t n, const void *hdr, size_t hlen, cudaStream_t st) {
    const uint64_t per = (uint64_t)P.max_windows * sizeof(DflNolzWin), fit = kDflNolzPassBytes / per;
    const uint32_t inputs = fit >= n ? n : (fit ? (uint32_t)fit : 1);
    Layout L;
    const size_t oWin = L.take((size_t)inputs * per), oHdr = L.take(hlen ? hlen : 1);
    { int r = reserve(ctx, ctx->d_dfl, L.end); if (r) return r; }
    { int r = ctx_order_begin(ctx, st); if (r) return r; }
    P.wins = ctx->d_dfl.at<DflNolzWin>(oWin);
    P.hdr = ctx->d_dfl.p + oHdr; P.hlen = (uint32_t)hlen;
    if (hlen) CK(cudaMemcpyAsync(ctx->d_dfl.p + oHdr, hdr, hlen, cudaMemcpyHostToDevice, st));
    const bool analyse = P.level != 0 || P.format != B2C_FLATE_RAW || P.crc_out;
    for (uint32_t i0 = 0; i0 < n; i0 += inputs) {
        P.i0 = i0; P.i1 = n - i0 < inputs ? n : i0 + inputs;
        const uint64_t slots = (uint64_t)(P.i1 - P.i0) * P.max_windows;
        if (analyse) b2c_deflate_nolz_analyse_kernel<<<(unsigned)slots, DFL_NOLZ_THREADS, 0, st>>>(P);
        b2c_deflate_nolz_plan_kernel<<<(P.i1 - P.i0 + DFL_NOLZ_PLAN_WARPS - 1) / DFL_NOLZ_PLAN_WARPS, DFL_NOLZ_PLAN_WARPS * 32, 0, st>>>(P);
        b2c_deflate_nolz_emit_kernel<<<(unsigned)slots, DFL_NOLZ_THREADS, 0, st>>>(P);
        ctx->launches += analyse ? 3 : 2;
        if (P.level != 0) {                            // level 0 is byte-aligned: no byte is shared
            b2c_deflate_nolz_finish_kernel<<<(unsigned)((slots + DFL_NOLZ_THREADS - 1) / DFL_NOLZ_THREADS), DFL_NOLZ_THREADS, 0, st>>>(P, slots);
            ctx->launches += 1;
        }
        CK(cudaGetLastError());
    }
    return ctx_order_end(ctx, st);
}

int b2c_flate_nolz_device(b2c_ctx *ctx, int level, int format, int flags, const void *d_src, size_t src_stride,
                          const uint64_t *d_src_offsets, const uint32_t *d_src_sizes, const void *hdr, size_t hlen,
                          void *d_dst, size_t dst_stride, const uint64_t *d_dst_offsets, uint32_t dst_cap,
                          int64_t *d_out_sizes, uint32_t *d_check_out, uint32_t nchunks, void *stream) {
    if (!ctx) return B2C_ERR_NO_DEVICE;
    if ((level != 0 && level != -2) || !best_speed_args_ok(format, flags, hdr, hlen)) return B2C_ERR_ARG;
    if (!d_src_sizes || !d_out_sizes || src_stride == 0 || src_stride > 0xffffffffull) return B2C_ERR_ARG;
    if (nchunks == 0) return B2C_OK;
    CK(cudaSetDevice(ctx->device));
    DflNolzParams P;
    memset(&P, 0, sizeof(P));
    P.src_base = (const uint8_t *)d_src; P.src_stride = src_stride; P.src_offsets = d_src_offsets; P.src_sizes = d_src_sizes;
    P.dst_base = (uint8_t *)d_dst; P.dst_stride = dst_stride; P.dst_offsets = d_dst_offsets; P.dst_cap = dst_cap;
    P.out_sizes = d_out_sizes; P.crc_out = d_check_out;
    P.format = format; P.level = level;
    P.max_windows = dfl_nolz_windows(src_stride, level);
    return launch_nolz(ctx, P, nchunks, hdr, hlen, (cudaStream_t)stream);
}

int b2c_flate_nolz_chunks(b2c_ctx *ctx, int level, int format, int flags, const void *const *srcs, const size_t *src_sizes,
                          const void *hdr, size_t hlen, void *const *dsts, const size_t *dst_caps, int64_t *sizes_out,
                          uint32_t *check_out, size_t n) {
    if (!ctx) return B2C_ERR_NO_DEVICE;
    if ((level != 0 && level != -2) || !best_speed_args_ok(format, flags, hdr, hlen)) return B2C_ERR_ARG;
    if (n == 0) return B2C_OK;
    int rc = HostBatch::check(ctx, n, src_sizes, 0xffffffffull);
    if (rc) return rc;
    HostBatch B(ctx, n, n, {n * 4});                                  // + the checksums
    B.place_items(src_sizes, 0, dst_caps, 0);
    uint32_t mw = 1;
    for (size_t i = 0; i < n; i++) {
        const uint32_t w = dfl_nolz_windows(src_sizes[i], level);
        if (w > mw) mw = w;
    }
    if ((rc = B.stage_in(srcs, src_sizes))) return rc;
    DflNolzParams P = B.params<DflNolzParams>();
    P.crc_out = B.d_at<uint32_t>(B.ex[0]);
    P.format = format; P.level = level; P.max_windows = mw;
    if ((rc = launch_nolz(ctx, P, (uint32_t)n, hdr, hlen, ctx->stream))) return rc;
    if (check_out) CK(cudaMemcpyAsync(check_out, P.crc_out, n * 4, cudaMemcpyDeviceToHost, ctx->stream));
    if ((rc = B.results(sizes_out))) return rc;
    return B.scatter(dsts, sizes_out, dst_caps);
}

// ---- standalone huff0 blocks ------------------------------------------------------------------------
int b2c_huf_compress_device(b2c_ctx *ctx, int flags, const void *d_src, size_t src_stride, const uint32_t *d_sizes,
                            uint32_t size_all, void *d_dst, size_t dst_stride, int64_t *d_out_sizes, uint32_t nchunks,
                            void *stream) {
    if (!ctx) return B2C_ERR_NO_DEVICE;
    if (nchunks == 0) return B2C_OK;
    if ((dst_stride & 3) || (reinterpret_cast<uintptr_t>(d_dst) & 3) || dst_stride > 0xffffffffull) return B2C_ERR_ARG;
    CK(cudaSetDevice(ctx->device));
    Huf0Params P;
    memset(&P, 0, sizeof(P));
    P.src_base = (const uint8_t *)d_src; P.src_stride = src_stride; P.src_sizes = d_sizes; P.src_size_all = size_all;
    P.dst_base = (uint8_t *)d_dst; P.dst_stride = dst_stride; P.dst_cap = (uint32_t)dst_stride;
    P.out_sizes = d_out_sizes; P.nchunks = nchunks; P.flags = (flags & B2C_HUF_4X) ? HUF0_FLAG_4X : 0;
    unsigned grid = (unsigned)ctx->sm_count * 2 < nchunks ? (unsigned)ctx->sm_count * 2 : nchunks;
    b2c_huf_compress_kernel<<<grid, HUF0_NT, HUF0_SMEM_BYTES, (cudaStream_t)stream>>>(P);
    ctx->launches += 1;
    CK(cudaGetLastError());
    return B2C_OK;
}

int b2c_huf_decompress_device(b2c_ctx *ctx, int flags, const void *d_src, size_t src_stride, const uint32_t *d_src_sizes,
                              void *d_dst, size_t dst_stride, const uint32_t *d_dst_sizes, int64_t *d_out_sizes,
                              uint32_t nchunks, void *stream) {
    if (!ctx) return B2C_ERR_NO_DEVICE;
    if (!d_src_sizes || !d_dst_sizes || !d_out_sizes) return B2C_ERR_ARG;
    if (nchunks == 0) return B2C_OK;
    CK(cudaSetDevice(ctx->device));
    Huf0Params P;
    memset(&P, 0, sizeof(P));
    P.src_base = (const uint8_t *)d_src; P.src_stride = src_stride; P.src_sizes = d_src_sizes;
    P.dst_base = (uint8_t *)d_dst; P.dst_stride = dst_stride; P.dst_sizes = d_dst_sizes;
    P.out_sizes = d_out_sizes; P.nchunks = nchunks; P.flags = (flags & B2C_HUF_4X) ? HUF0_FLAG_4X : 0;
    const unsigned grid = dec_grid(ctx, nchunks);
    cudaStream_t st = (cudaStream_t)stream;
    // Staged form (the default): table pass -> the staged zstd decoder's literal-stream kernel -> the one-warp kernel over what
    // is left (errors, unusual blocks).  B2C_DEC=onewarp, very large batches and unaligned slots keep the one-warp kernel alone.
    const bool staged = ctx->dec_staged && nchunks <= (1u << 20) && (dst_stride & 3) == 0;
    if (staged) {
        ctx->fd_last = false;           // the records below overwrite the zstd decoder's
        Layout L;
        const size_t oRec = L.take((size_t)nchunks * sizeof(FdChunk)), oBlk = L.take((size_t)nchunks * sizeof(FdBlock)),
                     oHuf = L.take((size_t)nchunks * 2048 * sizeof(uint16_t));
        { int r = ctx_order_begin(ctx, st); if (r) return r; }
        int rc = reserve(ctx, ctx->d_fd, L.end);
        if (rc) return rc;
        P.fd = ctx->d_fd.at<FdChunk>(oRec);
        P.fd_blk = ctx->d_fd.at<FdBlock>(oBlk);
        P.fd_huf = ctx->d_fd.at<uint16_t>(oHuf);
        b2c_huf_dec_prep_kernel<<<grid, DEC_WARPS * 32, DEC_SMEM_BYTES, st>>>(P);
        ZstdDecParams Z;
        memset(&Z, 0, sizeof(Z));
        Z.src_base = P.src_base; Z.src_stride = src_stride; Z.src_sizes = d_src_sizes;
        Z.dst_base = P.dst_base; Z.dst_stride = dst_stride; Z.out_sizes = d_out_sizes; Z.nchunks = nchunks;
        Z.fd = P.fd; Z.fd_blk = P.fd_blk; Z.fd_maxb = 1; Z.fd_per_block = 0; Z.fd_huf = P.fd_huf; Z.fd_lits = P.dst_base; Z.fd_lit_stride = dst_stride;
        const unsigned groups = (nchunks + FD_LIT_GROUP - 1) / FD_LIT_GROUP;
        b2c_zstd_dec_lit_kernel<<<(groups + FD_LIT_WARPS - 1) / FD_LIT_WARPS, FD_LIT_WARPS * 32, FD_LIT_WARPS * FD_LIT_WARP_BYTES, st>>>(Z);
        ctx->launches += 2;
    }
    b2c_huf_decompress_kernel<<<grid, DEC_WARPS * 32, DEC_SMEM_BYTES, st>>>(P);
    ctx->launches += 1;
    CK(cudaGetLastError());
    if (staged) return ctx_order_end(ctx, st);
    return B2C_OK;
}

// Host-buffer batches for the standalone huff0 calls (huff0.Compress4X / Compress1X, Decoder.Decompress4X / 1X, ReadTable
// per element): inputs are packed into equal slots on the device, one kernel per call, results copied back.
//   op 0: compress (dst_caps = capacities), op 1: decompress (dst_caps = EXACT decoded sizes), op 2: read table
//   (dsts[i] receives the 260-byte row described in include/b2c.h)
static int huf_host_batch(b2c_ctx *ctx, int op, int flags, const void *const *srcs, const size_t *src_sizes,
                          void *const *dsts, const size_t *dst_caps, int64_t *sizes_out, size_t n) {
    if (!ctx) return B2C_ERR_NO_DEVICE;
    if (n == 0) return B2C_OK;
    int rc = HostBatch::check(ctx, n, src_sizes, 0x7fffffffull);
    if (rc) return rc;
    size_t maxIn = 16, maxOut = 16;
    for (size_t i = 0; i < n; i++) {
        if (src_sizes[i] > maxIn) maxIn = src_sizes[i];
        const size_t want = op == 2 ? 260 : (op == 0 ? (dst_caps[i] < src_sizes[i] ? dst_caps[i] : src_sizes[i]) : dst_caps[i]);
        if (want > maxOut) maxOut = want;
    }
    if (op == 1 && maxOut > 262144) maxOut = 262144;      // larger exact sizes are refused by the kernel (ErrTooBig class)
    const size_t inStride = (maxIn + 15) & ~(size_t)15, outStride = (maxOut + 15) & ~(size_t)15;
    HostBatch B(ctx, n, n);
    B.place_items(src_sizes, inStride, dst_caps, outStride);
    if ((rc = B.stage_in(srcs, src_sizes))) return rc;
    uint8_t *d_in = ctx->d_dec_in.p, *d_out = ctx->d_dec_out.p;
    if (op == 0)
        rc = b2c_huf_compress_device(ctx, flags, d_in, inStride, B.d.src_sizes, 0, d_out, outStride, B.d.res, (uint32_t)n, ctx->stream);
    else if (op == 1)
        rc = b2c_huf_decompress_device(ctx, flags, d_in, inStride, B.d.src_sizes, d_out, outStride, B.d.dst_caps, B.d.res, (uint32_t)n,
                                       ctx->stream);
    else {
        Huf0Params P;
        memset(&P, 0, sizeof(P));
        P.src_base = d_in; P.src_stride = inStride; P.src_sizes = B.d.src_sizes;
        P.dst_base = d_out; P.dst_stride = outStride; P.out_sizes = B.d.res; P.nchunks = (uint32_t)n;
        b2c_huf_read_table_kernel<<<dec_grid(ctx, (uint32_t)n), DEC_WARPS * 32, DEC_SMEM_BYTES, ctx->stream>>>(P);
        ctx->launches += 1;
        CK(cudaGetLastError());
    }
    if (rc || (rc = B.results(sizes_out))) return rc;
    return B.scatter(dsts, sizes_out, dst_caps, op == 2 ? 260 : 0);
}
int b2c_huf_compress_chunks(b2c_ctx *ctx, int flags, const void *const *srcs, const size_t *src_sizes, void *const *dsts,
                            const size_t *dst_caps, int64_t *sizes_out, size_t n) {
    return huf_host_batch(ctx, 0, flags, srcs, src_sizes, dsts, dst_caps, sizes_out, n);
}
int b2c_huf_decompress_chunks(b2c_ctx *ctx, int flags, const void *const *srcs, const size_t *src_sizes, void *const *dsts,
                              const size_t *dst_sizes, int64_t *sizes_out, size_t n) {
    return huf_host_batch(ctx, 1, flags, srcs, src_sizes, dsts, dst_sizes, sizes_out, n);
}
int b2c_huf_read_table(b2c_ctx *ctx, const void *const *srcs, const size_t *src_sizes, void *const *rows, int64_t *sizes_out, size_t n) {
    std::vector<size_t> caps(n, 260);
    return huf_host_batch(ctx, 2, 0, srcs, src_sizes, rows, caps.data(), sizes_out, n);
}

// ---- coalescing queue ---------------------------------------------------------------------------------------------
// The reference's seams are one block per call from many goroutines at once: zstd.Encoder.EncodeAll "can be called
// concurrently" (zstd/encoder.go:717-729), s2.WriterCustomEncoder's hook runs on one goroutine per block
// (s2/writer.go:1052-1064, call sites :455-461), Decoder.DecodeAll likewise.  A GPU wants batches.  b2c_queue is the
// piece of the shim that turns the former into the latter: callers block in b2c_queue_*; one dispatcher thread owns
// the context, collects what is pending (lingering a few microseconds for stragglers), issues ONE *_chunks call per
// kind of request and wakes the callers with their results.  Caller memory is only touched during the call.
struct b2c_req {
    int op, level, flags;                 // op: 0 zstd encode, 1 s2 encode, 2 zstd decode, 3 s2 decode
    const void *src; size_t n; void *dst; size_t cap;
    int64_t result; bool done;
};
struct b2c_queue {
    b2c_ctx *ctx = nullptr;
    size_t max_batch = 0;
    unsigned linger_us = 0;
    std::mutex mu;
    std::condition_variable cv_work, cv_done;
    std::deque<b2c_req *> pending;
    bool stop = false;
    std::thread worker;
    std::atomic<uint64_t> calls{0}, batches{0};
};

static void queue_run_batch(b2c_queue *q, std::vector<b2c_req *> &grp) {
    const size_t m = grp.size();
    std::vector<const void *> srcs(m);
    std::vector<void *> dsts(m);
    std::vector<size_t> ssz(m), dcap(m);
    std::vector<int64_t> res(m, 0);
    for (size_t i = 0; i < m; i++) { srcs[i] = grp[i]->src; ssz[i] = grp[i]->n; dsts[i] = grp[i]->dst; dcap[i] = grp[i]->cap; }
    const b2c_req *r0 = grp[0];
    int rc;
    switch (r0->op) {
    case 0: {
        // EncodeAll: inputs of at most one block are single-block frames (encode_chunks); larger ones go through frame mode
        // (one multi-block frame each), both as one device batch
        const size_t blk = level_ok(r0->level) ? level_block(r0->level) : 0;
        std::vector<size_t> big, small;
        for (size_t i = 0; i < m; i++) (ssz[i] > blk ? big : small).push_back(i);
        rc = B2C_OK;
        for (int pass = 0; pass < 2 && rc == B2C_OK; pass++) {
            const std::vector<size_t> &ix = pass ? big : small;
            if (ix.empty()) continue;
            const size_t k = ix.size();
            std::vector<const void *> s2(k); std::vector<void *> d2(k); std::vector<size_t> z2(k), c2(k); std::vector<int64_t> r2(k, 0);
            for (size_t j = 0; j < k; j++) { s2[j] = srcs[ix[j]]; d2[j] = dsts[ix[j]]; z2[j] = ssz[ix[j]]; c2[j] = dcap[ix[j]]; }
            rc = pass ? b2c_zstd_encode_frames(q->ctx, r0->level, r0->flags & B2C_ZSTD_CRC, s2.data(), z2.data(), d2.data(), c2.data(), r2.data(), k)
                      : b2c_zstd_encode_chunks(q->ctx, r0->level, r0->flags, s2.data(), z2.data(), d2.data(), c2.data(), r2.data(), k);
            for (size_t j = 0; j < k; j++) res[ix[j]] = r2[j];
        }
        break;
    }
    case 1: rc = b2c_s2_encode_chunks(q->ctx, r0->level, r0->flags, srcs.data(), ssz.data(), dsts.data(), dcap.data(), res.data(), m); break;
    case 2: rc = b2c_zstd_decode_chunks(q->ctx, srcs.data(), ssz.data(), dsts.data(), dcap.data(), res.data(), m); break;
    default: rc = b2c_s2_decode_chunks(q->ctx, srcs.data(), ssz.data(), dsts.data(), dcap.data(), res.data(), m); break;
    }
    for (size_t i = 0; i < m; i++) grp[i]->result = rc ? (int64_t)rc : res[i];
    q->batches++;
}

static void queue_worker(b2c_queue *q) {
    cudaSetDevice(q->ctx->device);
    std::unique_lock<std::mutex> lk(q->mu);
    for (;;) {
        q->cv_work.wait(lk, [&] { return q->stop || !q->pending.empty(); });
        if (q->pending.empty()) { if (q->stop) return; continue; }
        if (q->linger_us && q->pending.size() < q->max_batch && !q->stop)   // give concurrent callers a moment to arrive
            q->cv_work.wait_for(lk, std::chrono::microseconds(q->linger_us), [&] { return q->stop || q->pending.size() >= q->max_batch; });
        std::vector<b2c_req *> take;
        while (!q->pending.empty() && take.size() < q->max_batch) { take.push_back(q->pending.front()); q->pending.pop_front(); }
        lk.unlock();
        // one device batch per kind of request, in arrival order of the kinds
        std::vector<char> used(take.size(), 0);
        for (size_t i = 0; i < take.size(); i++) {
            if (used[i]) continue;
            std::vector<b2c_req *> grp;
            for (size_t j = i; j < take.size(); j++)
                if (!used[j] && take[j]->op == take[i]->op && take[j]->level == take[i]->level && take[j]->flags == take[i]->flags) {
                    grp.push_back(take[j]); used[j] = 1;
                }
            queue_run_batch(q, grp);
        }
        lk.lock();
        for (b2c_req *r : take) r->done = true;
        q->cv_done.notify_all();
    }
}

static int64_t queue_call(b2c_queue *q, int op, int level, int flags, const void *src, size_t n, void *dst, size_t cap) {
    if (!q) return B2C_ERR_NO_DEVICE;
    b2c_req r{op, level, flags, src, n, dst, cap, 0, false};
    std::unique_lock<std::mutex> lk(q->mu);
    if (q->stop) return B2C_ERR_ARG;
    q->pending.push_back(&r);
    q->calls++;
    q->cv_work.notify_one();
    q->cv_done.wait(lk, [&] { return r.done; });
    return r.result;
}

b2c_queue *b2c_queue_create(int device, size_t max_batch, unsigned linger_us) {
    if (max_batch == 0) max_batch = 1024;
    b2c_ctx *ctx = b2c_ctx_create(device, max_batch);
    if (!ctx) return nullptr;
    b2c_queue *q = new b2c_queue();
    q->ctx = ctx; q->max_batch = max_batch; q->linger_us = linger_us;
    q->worker = std::thread(queue_worker, q);
    return q;
}
void b2c_queue_destroy(b2c_queue *q) {
    if (!q) return;
    { std::lock_guard<std::mutex> lk(q->mu); q->stop = true; }
    q->cv_work.notify_all();
    if (q->worker.joinable()) q->worker.join();
    b2c_ctx_destroy(q->ctx);
    delete q;
}
int64_t b2c_queue_zstd_encode(b2c_queue *q, int level, int flags, const void *src, size_t n, void *dst, size_t cap) {
    return queue_call(q, 0, level, flags, src, n, dst, cap);
}
int64_t b2c_queue_s2_encode(b2c_queue *q, int level, int flags, const void *src, size_t n, void *dst, size_t cap) {
    return queue_call(q, 1, level, flags, src, n, dst, cap);
}
int64_t b2c_queue_zstd_decode(b2c_queue *q, const void *src, size_t n, void *dst, size_t cap) {
    return queue_call(q, 2, 0, 0, src, n, dst, cap);
}
int64_t b2c_queue_s2_decode(b2c_queue *q, const void *src, size_t n, void *dst, size_t cap) {
    return queue_call(q, 3, 0, 0, src, n, dst, cap);
}
int b2c_queue_stats(b2c_queue *q, uint64_t *calls, uint64_t *batches) {
    if (!q) return B2C_ERR_NO_DEVICE;
    if (calls) *calls = q->calls.load();
    if (batches) *batches = q->batches.load();
    return B2C_OK;
}

}  // extern "C"
