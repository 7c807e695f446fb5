// owshen_b200/csrc/capi.cu -- the extern "C" boundary declared in include/owshen_b200.h.
// Host-pointer entry points stage their buffers in persistent device slots (H2D/D2H on the ctx
// stream, truly asynchronous when the caller's memory is pinned) and return after the result has
// landed; `_dev` entry points only enqueue.  No entry point has a CPU implementation.
#include <stdlib.h>
#include <new>
#include "common.cuh"
#include "groth16.cuh"
#include "mimc.cuh"
#include "msm.cuh"
#include "ntt.cuh"
#include "withdraw_circuit.hpp"

using namespace og;

void* og_ctx::slot(int id, size_t bytes) {
    if (bytes == 0) bytes = 32;
    if (slot_cap[id] >= bytes) return slot_ptr[id];
    cudaDeviceSynchronize();          // growth is rare; other lanes may still be using neighbouring slots' kernels
    if (slot_ptr[id]) cudaFree(slot_ptr[id]);
    slot_ptr[id] = nullptr; slot_cap[id] = 0;
    size_t cap = bytes + bytes / 8;
    cudaError_t e = cudaMalloc(&slot_ptr[id], cap);
    if (e != cudaSuccess) {
        e = cudaMalloc(&slot_ptr[id], bytes);
        cap = bytes;
    }
    if (e != cudaSuccess) {
        snprintf(err, sizeof(err), "slot %d: cudaMalloc(%zu) failed: %s", id, bytes, cudaGetErrorString(e));
        slot_ptr[id] = nullptr;
        return nullptr;
    }
    slot_cap[id] = cap;
    return slot_ptr[id];
}

cudaEvent_t og_ctx::prof_event() {
    if (!ev_pool.empty()) { cudaEvent_t e = ev_pool.back(); ev_pool.pop_back(); return e; }
    cudaEvent_t e = nullptr;
    cudaEventCreate(&e);
    return e;
}

namespace og {
int32_t clear_flag(og_ctx* ctx) {
    OG_CUDA(ctx, cudaMemsetAsync(ctx->d_flag, 0, sizeof(int), ctx->stream));
    return OG_OK;
}
int32_t check_flag(og_ctx* ctx) {
    OG_CUDA(ctx, cudaMemcpyAsync(ctx->h_flag, ctx->d_flag, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    OG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (*ctx->h_flag) { snprintf(ctx->err, sizeof(ctx->err), "non-canonical field element in input"); return OG_E_ENCODING; }
    return OG_OK;
}
}  // namespace og

// every entry point that takes a ctx first makes its device current: several contexts (one per GPU) may live in
// one process (INTEGRATION.md: one Prover per GPU), and launches go to the calling thread's current device
#define OG_ENTER(ctx)                                                                              \
    do {                                                                                           \
        if (!(ctx)) return OG_E_INVALID;                                                           \
        OG_CUDA(ctx, cudaSetDevice((ctx)->device));                                                \
    } while (0)

// a proving key's tables are device memory of the GPU it was loaded on: refuse it on any other context's GPU
#define OG_PK_CHECK(ctx, pk)                                                                           \
    do {                                                                                               \
        if (!pk_on_device_of(pk, ctx)) {                                                               \
            snprintf((ctx)->err, sizeof((ctx)->err), "proving key was loaded on another device");      \
            return OG_E_INVALID;                                                                       \
        }                                                                                              \
    } while (0)

#define H2D(ctx, dst, src, bytes) OG_CUDA(ctx, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, (ctx)->stream))
#define D2H(ctx, dst, src, bytes) OG_CUDA(ctx, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, (ctx)->stream))

extern "C" {

int32_t og_abi_version(void) { return 1; }

const char* og_strerror(int32_t code) {
    switch (code) {
        case OG_OK: return "ok";
        case OG_E_INVALID: return "invalid argument";
        case OG_E_ENCODING: return "malformed or non-canonical encoding";
        case OG_E_NO_DEVICE: return "no usable CUDA device (this library has no CPU path)";
        case OG_E_CUDA: return "CUDA runtime error";
        case OG_E_NOMEM: return "out of device memory";
        case OG_E_VERIFY: return "proof does not verify";
        default: return "unknown error";
    }
}
const char* og_last_error(const og_ctx* ctx) { return ctx ? ctx->err : ""; }

int32_t og_init(int32_t device, og_ctx** out) {
    if (!out) return OG_E_INVALID;
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0 || device < 0 || device >= n) return OG_E_NO_DEVICE;
    if (cudaSetDevice(device) != cudaSuccess) return OG_E_NO_DEVICE;
    og_ctx* ctx = new og_ctx();
    ctx->device = device;
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) ctx->sm_count = prop.multiProcessorCount;
    if (cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) != cudaSuccess ||
        cudaEventCreate(&ctx->ev0) != cudaSuccess || cudaEventCreate(&ctx->ev1) != cudaSuccess ||
        cudaMalloc(&ctx->d_flag, sizeof(int)) != cudaSuccess || cudaMallocHost(&ctx->h_flag, sizeof(int)) != cudaSuccess) {
        delete ctx;
        return OG_E_CUDA;
    }
    cudaMemset(ctx->d_flag, 0, sizeof(int));
    ctx->main_stream = ctx->stream;
    {
        int least = 0, greatest = 0;
        cudaDeviceGetStreamPriorityRange(&least, &greatest);
        { const char* v = getenv("OG_LANE_PRIO"); if (v && atoi(v) == 0) least = greatest = 0; }   // A/B: lanes without stream priorities
        bool ok = cudaEventCreateWithFlags(&ctx->fork_ev, cudaEventDisableTiming) == cudaSuccess &&
                  cudaEventCreateWithFlags(&ctx->acc_ev, cudaEventDisableTiming) == cudaSuccess;
        for (int l = 0; ok && l < MAX_LANES; l++)
            ok = cudaStreamCreateWithPriority(&ctx->lane_hi[l], cudaStreamNonBlocking, greatest) == cudaSuccess &&
                 cudaStreamCreateWithPriority(&ctx->lane_lo[l], cudaStreamNonBlocking, least) == cudaSuccess &&
                 cudaEventCreateWithFlags(&ctx->lane_ev[l], cudaEventDisableTiming) == cudaSuccess;
        if (!ok) { og_free(ctx); return OG_E_CUDA; }
    }
    int32_t rc = mimc_init(ctx);
    if (rc != OG_OK) { og_free(ctx); return rc; }
    *out = ctx;
    return OG_OK;
}

void og_free(og_ctx* ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    cudaDeviceSynchronize();
    ctx->stream = ctx->main_stream ? ctx->main_stream : ctx->stream;
    for (int l = 0; l < MAX_LANES; l++) {
        if (ctx->lane_hi[l]) cudaStreamDestroy(ctx->lane_hi[l]);
        if (ctx->lane_lo[l]) cudaStreamDestroy(ctx->lane_lo[l]);
        if (ctx->lane_ev[l]) cudaEventDestroy(ctx->lane_ev[l]);
    }
    if (ctx->fork_ev) cudaEventDestroy(ctx->fork_ev);
    if (ctx->acc_ev) cudaEventDestroy(ctx->acc_ev);
    for (int i = 0; i < N_SLOTS; i++) if (ctx->slot_ptr[i]) cudaFree(ctx->slot_ptr[i]);
    ntt_free_tables(ctx);
    if (ctx->g1_fixed) cudaFree(ctx->g1_fixed);
    if (ctx->g2_fixed) cudaFree(ctx->g2_fixed);
    if (ctx->bjj_fixed) cudaFree(ctx->bjj_fixed);
    if (ctx->d_flag) cudaFree(ctx->d_flag);
    if (ctx->h_flag) cudaFreeHost(ctx->h_flag);
    for (auto& r : ctx->prof) { cudaEventDestroy(r.a); cudaEventDestroy(r.b); }
    for (auto e : ctx->ev_pool) cudaEventDestroy(e);
    if (ctx->ev0) cudaEventDestroy(ctx->ev0);
    if (ctx->ev1) cudaEventDestroy(ctx->ev1);
    if (ctx->stream) cudaStreamDestroy(ctx->stream);
    delete ctx;
}

int32_t og_sync(og_ctx* ctx) {
    OG_ENTER(ctx);
    if (!ctx) return OG_E_INVALID;
    OG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return OG_OK;
}
int32_t og_stream(og_ctx* ctx, void** out_cuda_stream) {
    if (!ctx || !out_cuda_stream) return OG_E_INVALID;
    *out_cuda_stream = (void*)ctx->main_stream;
    return OG_OK;
}
int32_t og_timer_start(og_ctx* ctx) {
    OG_ENTER(ctx);
    if (!ctx) return OG_E_INVALID;
    OG_CUDA(ctx, cudaEventRecord(ctx->ev0, ctx->stream));
    return OG_OK;
}
int32_t og_timer_stop(og_ctx* ctx, float* ms) {
    OG_ENTER(ctx);
    if (!ctx || !ms) return OG_E_INVALID;
    OG_CUDA(ctx, cudaEventRecord(ctx->ev1, ctx->stream));
    OG_CUDA(ctx, cudaEventSynchronize(ctx->ev1));
    OG_CUDA(ctx, cudaEventElapsedTime(ms, ctx->ev0, ctx->ev1));
    return OG_OK;
}
uint64_t og_launch_count(const og_ctx* ctx) { return ctx ? ctx->launches : 0; }

int32_t og_profile(og_ctx* ctx, int32_t enable) {
    OG_ENTER(ctx);
    if (!ctx) return OG_E_INVALID;
    ctx->prof_on = enable != 0;
    return OG_OK;
}
// "name,launches,total_ms\n" per kernel since the last dump; synchronises the stream
int32_t og_profile_dump(og_ctx* ctx, char* buf, uint64_t cap) {
    OG_ENTER(ctx);
    if (!ctx || !buf || cap == 0) return OG_E_INVALID;
    OG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    struct Agg { const char* name; uint64_t n; double ms; };
    std::vector<Agg> agg;
    for (auto& r : ctx->prof) {
        float ms = 0;
        cudaEventElapsedTime(&ms, r.a, r.b);
        size_t k = 0;
        for (; k < agg.size(); k++) if (strcmp(agg[k].name, r.name) == 0) break;
        if (k == agg.size()) agg.push_back({r.name, 0, 0.0});
        agg[k].n++; agg[k].ms += ms;
        ctx->ev_pool.push_back(r.a); ctx->ev_pool.push_back(r.b);
    }
    ctx->prof.clear();
    uint64_t off = 0;
    buf[0] = 0;
    for (auto& a : agg) {
        int w = snprintf(buf + off, cap - off, "%s,%llu,%.6f\n", a.name, (unsigned long long)a.n, a.ms);
        if (w < 0 || (uint64_t)w >= cap - off) break;
        off += (uint64_t)w;
    }
    return OG_OK;
}

// ---- field probes --------------------------------------------------------------------------------------
}  // extern "C"

namespace og {
template <class F>
__global__ void __launch_bounds__(128) k_field_op(int op, const uint8_t* __restrict__ a, const uint8_t* __restrict__ b, uint64_t n,
                                                  uint8_t* __restrict__ out, int* flag) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    F x = load_canonical<F>(a + 32 * i, flag), y = load_canonical<F>(b + 32 * i, flag);
    F r = op == 0 ? x * y : (op == 1 ? x + y : x - y);
    store_canonical(out + 32 * i, r);
}

// integer-pipe micro-benchmark.  Every multiply-add takes its own accumulator as a multiplicand, so ptxas
// cannot hoist the product out of the loop (an earlier version with loop-invariant multiplicands was
// strength-reduced to additions and measured the ALU pipe instead).  MODE 0: mad.lo.u32 (IMAD),
// MODE 1: mad.wide.u32 (IMAD.WIDE), MODE 2: mad.lo.cc/madc.hi.cc pairs in 4-pair carry chains, the
// shape of one Montgomery row (IMAD.WIDE.U32.X); a pair counts as ONE 32x32->64 multiply-add.
template <int MODE>
__global__ void __launch_bounds__(256) k_imad(uint32_t* out, uint32_t iters, uint32_t seed) {
    uint32_t x = blockIdx.x * 2654435761u + 12345u + seed, y = x ^ 0x9e3779b9u;
    if (MODE == 0) {
        uint32_t w[8];
#pragma unroll
        for (int k = 0; k < 8; k++) w[k] = threadIdx.x * (2 * k + 3) + seed;
        for (uint32_t i = 0; i < iters; i++) {
#pragma unroll
            for (int r = 0; r < 8; r++)
#pragma unroll
                for (int k = 0; k < 8; k++) asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(w[k]) : "r"(x), "r"(y));
        }
        uint32_t s = 0;
#pragma unroll
        for (int k = 0; k < 8; k++) s ^= w[k];
        if (s == 0x1234567u) out[0] = s;
    } else if (MODE == 1) {
        unsigned long long w[8];
#pragma unroll
        for (int k = 0; k < 8; k++) w[k] = threadIdx.x * (2 * k + 3) + seed;
        for (uint32_t i = 0; i < iters; i++) {
#pragma unroll
            for (int r = 0; r < 8; r++)
#pragma unroll
                for (int k = 0; k < 8; k++) {
                    uint32_t lo = (uint32_t)w[k];
                    asm volatile("mad.wide.u32 %0, %1, %2, %0;" : "+l"(w[k]) : "r"(lo), "r"(x));
                }
        }
        unsigned long long s = 0;
#pragma unroll
        for (int k = 0; k < 8; k++) s ^= w[k];
        if (s == 0x1234567ull) out[0] = (uint32_t)s;
    } else {
        uint32_t e[8], o[8];
#pragma unroll
        for (int k = 0; k < 8; k++) { e[k] = threadIdx.x * (2 * k + 3) + seed; o[k] = e[k] ^ y; }
        CC cc;
        for (uint32_t i = 0; i < iters; i++) {
#pragma unroll
            for (int r = 0; r < 4; r++) {
                uint32_t m0 = e[7] | 1u, m1 = o[7] | 1u;      // multiplicand depends on the previous chain
                e[0] = mad_lo_cc(m0, x, e[0], cc); e[1] = madc_hi_cc(m0, x, e[1], cc);
                e[2] = madc_lo_cc(m0, y, e[2], cc); e[3] = madc_hi_cc(m0, y, e[3], cc);
                e[4] = madc_lo_cc(m0, x, e[4], cc); e[5] = madc_hi_cc(m0, x, e[5], cc);
                e[6] = madc_lo_cc(m0, y, e[6], cc); e[7] = madc_hi(m0, y, e[7], cc);
                o[0] = mad_lo_cc(m1, x, o[0], cc); o[1] = madc_hi_cc(m1, x, o[1], cc);
                o[2] = madc_lo_cc(m1, y, o[2], cc); o[3] = madc_hi_cc(m1, y, o[3], cc);
                o[4] = madc_lo_cc(m1, x, o[4], cc); o[5] = madc_hi_cc(m1, x, o[5], cc);
                o[6] = madc_lo_cc(m1, y, o[6], cc); o[7] = madc_hi(m1, y, o[7], cc);
            }
        }
        uint32_t s = 0;
#pragma unroll
        for (int k = 0; k < 8; k++) s ^= e[k] ^ o[k];
        if (s == 0x1234567u) out[0] = s;
    }
}
// latency probe: cycles per DEPENDENT Montgomery multiplication for one warp alone on its scheduler
// (the MiMC chains are exactly this), and with two independent chains interleaved
template <int CHAINS>
__global__ void __launch_bounds__(32) k_mul_latency(Fr* io, uint32_t iters, long long* cycles) {
    Fr x = io[threadIdx.x], y = io[32 + threadIdx.x], k = io[64 + threadIdx.x];
    long long t0 = clock64();
    for (uint32_t i = 0; i < iters; i++) {
        x = x * x + k;
        if (CHAINS == 2) y = y * y + k;
    }
    long long t1 = clock64();
    io[threadIdx.x] = x + y;
    if (threadIdx.x == 0 && blockIdx.x == 0) cycles[0] = (t1 - t0);
}

// FP64 pipe probe (round-2 planning: DFMA-based 52-bit-limb products would run beside the integer pipe)
__global__ void __launch_bounds__(256) k_dfma(double* out, uint32_t iters, double seed) {
    double w[8], x = 1.0000001 + seed * 1e-9, y = 0.9999999;
#pragma unroll
    for (int k = 0; k < 8; k++) w[k] = threadIdx.x * 0.001 + k + seed;
    for (uint32_t i = 0; i < iters; i++) {
#pragma unroll
        for (int r = 0; r < 8; r++)
#pragma unroll
            for (int k = 0; k < 8; k++) w[k] = __fma_rz(w[k], x, y);
    }
    double s = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) s += w[k];
    if (s == 1.2345) out[0] = s;
}

// Hybrid-multiplier probe (round-2 planning).  A 52x52-bit product on the FP64 pipe costs two DFMA, one DADD and
// two 64-bit integer adds (Emmart et al.: hi = fma_rz(a, b, 2^104), lo = fma_rz(a, b, 2^104 + 2^52 - hi), the bit
// patterns accumulate as integers).  MODE 0: those products alone; MODE 1: the carry-chain IMAD.WIDE rows alone;
// MODE 2: both interleaved in every warp -- does the chip run the two multipliers at the same time?
template <int MODE>
__global__ void __launch_bounds__(256) k_hybrid(unsigned long long* out, uint32_t iters, uint32_t seed) {
    const double C1 = 20282409603651670423947251286016.0;                  // 2^104
    const double C2 = 20282409603651670423947251286016.0 + 4503599627370496.0;   // 2^104 + 2^52
    double a[4], b[4];
    long long acc_hi[4] = {0, 0, 0, 0}, acc_lo[4] = {0, 0, 0, 0};
    uint32_t e[8], o[8];
    uint32_t x = blockIdx.x * 2654435761u + 12345u + seed, y = x ^ 0x9e3779b9u;
#pragma unroll
    for (int k = 0; k < 4; k++) { a[k] = (double)((threadIdx.x * 977u + k * 131u + seed) & 0xFFFFF) + 4503599627370.0; b[k] = a[k] * 0.5 + 7.0; }
#pragma unroll
    for (int k = 0; k < 8; k++) { e[k] = threadIdx.x * (2 * k + 3) + seed; o[k] = e[k] ^ y; }
    CC cc;
    for (uint32_t i = 0; i < iters; i++) {
#pragma unroll
        for (int r = 0; r < 4; r++) {
            if (MODE == 0 || MODE == 2) {
#pragma unroll
                for (int k = 0; k < 4; k++) {                                 // 4 products of 52 x 52 bits
                    double hi = __fma_rz(a[k], b[(k + r) & 3], C1);
                    double sub = C2 - hi;
                    double lo = __fma_rz(a[k], b[(k + r) & 3], sub);
                    acc_hi[k] += __double_as_longlong(hi);
                    acc_lo[k] += __double_as_longlong(lo);
                }
                a[r] = a[r] + 1.0;                                            // keep the products loop-variant
            }
            if (MODE == 1 || MODE == 2) {                                     // 8 products of 32 x 32 -> 64 bits (lo and hi halves fuse)
                uint32_t m0 = e[7] | 1u, m1 = o[7] | 1u;
                e[0] = mad_lo_cc(m0, x, e[0], cc); e[1] = madc_hi_cc(m0, x, e[1], cc);
                e[2] = madc_lo_cc(m0, y, e[2], cc); e[3] = madc_hi_cc(m0, y, e[3], cc);
                e[4] = madc_lo_cc(m0, x, e[4], cc); e[5] = madc_hi_cc(m0, x, e[5], cc);
                e[6] = madc_lo_cc(m0, y, e[6], cc); e[7] = madc_hi(m0, y, e[7], cc);
                o[0] = mad_lo_cc(m1, x, o[0], cc); o[1] = madc_hi_cc(m1, x, o[1], cc);
                o[2] = madc_lo_cc(m1, y, o[2], cc); o[3] = madc_hi_cc(m1, y, o[3], cc);
                o[4] = madc_lo_cc(m1, x, o[4], cc); o[5] = madc_hi_cc(m1, x, o[5], cc);
                o[6] = madc_lo_cc(m1, y, o[6], cc); o[7] = madc_hi(m1, y, o[7], cc);
            }
        }
    }
    unsigned long long s = 0;
#pragma unroll
    for (int k = 0; k < 4; k++) s ^= (unsigned long long)acc_hi[k] ^ (unsigned long long)acc_lo[k];
#pragma unroll
    for (int k = 0; k < 8; k++) s ^= e[k] ^ o[k];
    if (s == 0x1234567ull) out[0] = s;
}

}  // namespace og

extern "C" {

// rates[0] = 52x52 FP64-pipe products/s alone, rates[1] = 32x32->64 carry-chain IMAD.WIDE/s alone,
// rates[2], rates[3] = the same two rates when both run interleaved in every warp
int32_t og_hybrid_probe(og_ctx* ctx, double* rates4) {
    OG_ENTER(ctx);
    if (!rates4) return OG_E_INVALID;
    OG_SLOT(ctx, d_out, unsigned long long, S_IO_A, 64);
    const uint32_t iters = 1024, ctas = ctx->sm_count * 8, threads = 256;
    const double lanes = (double)ctas * threads * iters * 4.0;        // 4 rounds per iteration
    float ms[3] = {0, 0, 0};
    for (int mode = 0; mode < 3; mode++) {
        float best = 1e30f, t = 0;
        for (int rep = 0; rep < 4; rep++) {
            OG_CUDA(ctx, cudaEventRecord(ctx->ev0, ctx->stream));
            if (mode == 0) OG_LAUNCH(ctx, k_hybrid<0>, ctas, threads, 0, d_out, iters, (uint32_t)rep);
            else if (mode == 1) OG_LAUNCH(ctx, k_hybrid<1>, ctas, threads, 0, d_out, iters, (uint32_t)rep);
            else OG_LAUNCH(ctx, k_hybrid<2>, ctas, threads, 0, d_out, iters, (uint32_t)rep);
            OG_CUDA(ctx, cudaEventRecord(ctx->ev1, ctx->stream));
            OG_CUDA(ctx, cudaEventSynchronize(ctx->ev1));
            OG_CUDA(ctx, cudaEventElapsedTime(&t, ctx->ev0, ctx->ev1));
            if (rep > 0 && t < best) best = t;
        }
        ms[mode] = best;
    }
    rates4[0] = lanes * 4.0 / (ms[0] * 1e-3);
    rates4[1] = lanes * 8.0 / (ms[1] * 1e-3);      // lo+hi of one product fuse into one IMAD.WIDE
    rates4[2] = lanes * 4.0 / (ms[2] * 1e-3);
    rates4[3] = lanes * 8.0 / (ms[2] * 1e-3);
    return OG_OK;
}

int32_t og_mul_latency(og_ctx* ctx, double* cycles_dependent, double* cycles_two_chains) {
    OG_ENTER(ctx);
    if (!ctx || !cycles_dependent || !cycles_two_chains) return OG_E_INVALID;
    OG_SLOT(ctx, io, Fr, S_IO_A, sizeof(Fr) * 96 + 64);
    long long* d_cyc = reinterpret_cast<long long*>(io + 96);
    OG_CUDA(ctx, cudaMemsetAsync(io, 1, sizeof(Fr) * 96, ctx->stream));
    const uint32_t iters = 20000;
    long long h = 0;
    OG_LAUNCH(ctx, k_mul_latency<1>, 1, 32, 0, io, iters, d_cyc);
    OG_CUDA(ctx, cudaMemcpyAsync(&h, d_cyc, 8, cudaMemcpyDeviceToHost, ctx->stream));
    OG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    *cycles_dependent = (double)h / iters;
    OG_LAUNCH(ctx, k_mul_latency<2>, 1, 32, 0, io, iters, d_cyc);
    OG_CUDA(ctx, cudaMemcpyAsync(&h, d_cyc, 8, cudaMemcpyDeviceToHost, ctx->stream));
    OG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    *cycles_two_chains = (double)h / iters;
    return OG_OK;
}

int32_t og_fp64_peak(og_ctx* ctx, double* dfma_per_s) {
    OG_ENTER(ctx);
    if (!ctx || !dfma_per_s) return OG_E_INVALID;
    OG_SLOT(ctx, d_out, double, S_IO_A, 64);
    const uint32_t iters = 2048, ctas = ctx->sm_count * 8, threads = 256;
    float ms = 0;
    double best = 0;
    for (int rep = 0; rep < 4; rep++) {
        OG_CUDA(ctx, cudaEventRecord(ctx->ev0, ctx->stream));
        OG_LAUNCH(ctx, k_dfma, ctas, threads, 0, d_out, iters, (double)rep);
        OG_CUDA(ctx, cudaEventRecord(ctx->ev1, ctx->stream));
        OG_CUDA(ctx, cudaEventSynchronize(ctx->ev1));
        OG_CUDA(ctx, cudaEventElapsedTime(&ms, ctx->ev0, ctx->ev1));
        double rate = (double)ctas * threads * iters * 64.0 / (ms * 1e-3);
        if (rep > 0 && rate > best) best = rate;
    }
    *dfma_per_s = best;
    return OG_OK;
}

int32_t og_imad_peak(og_ctx* ctx, double* mad_per_s, double* wide_mad_per_s) {
    OG_ENTER(ctx);
    if (!ctx || !mad_per_s || !wide_mad_per_s) return OG_E_INVALID;
    double chain = 0;
    return og_int_pipe_peaks(ctx, mad_per_s, wide_mad_per_s, &chain);
}

int32_t og_int_pipe_peaks(og_ctx* ctx, double* mad_per_s, double* wide_mad_per_s, double* carry_chain_wide_per_s) {
    OG_ENTER(ctx);
    if (!ctx || !mad_per_s || !wide_mad_per_s || !carry_chain_wide_per_s) return OG_E_INVALID;
    OG_SLOT(ctx, d_out, uint32_t, S_IO_A, 64);
    const uint32_t iters = 2048, ctas = ctx->sm_count * 8, threads = 256;
    float ms = 0;
    double* outs[3] = {mad_per_s, wide_mad_per_s, carry_chain_wide_per_s};
    const double per_iter[3] = {64.0, 64.0, 32.0};
    for (int mode = 0; mode < 3; mode++) {
        double best = 0;
        for (int rep = 0; rep < 4; rep++) {
            OG_CUDA(ctx, cudaEventRecord(ctx->ev0, ctx->stream));
            if (mode == 0) OG_LAUNCH(ctx, k_imad<0>, ctas, threads, 0, d_out, iters, (uint32_t)rep);
            else if (mode == 1) OG_LAUNCH(ctx, k_imad<1>, ctas, threads, 0, d_out, iters, (uint32_t)rep);
            else OG_LAUNCH(ctx, k_imad<2>, ctas, threads, 0, d_out, iters, (uint32_t)rep);
            OG_CUDA(ctx, cudaEventRecord(ctx->ev1, ctx->stream));
            OG_CUDA(ctx, cudaEventSynchronize(ctx->ev1));
            OG_CUDA(ctx, cudaEventElapsedTime(&ms, ctx->ev0, ctx->ev1));
            double rate = (double)ctas * threads * iters * per_iter[mode] / (ms * 1e-3);
            if (rep > 0 && rate > best) best = rate;
        }
        *outs[mode] = best;
    }
    return OG_OK;
}

int32_t og_field_op(og_ctx* ctx, int32_t field, int32_t op, const uint8_t* a, const uint8_t* b, uint64_t n, uint8_t* out) {
    OG_ENTER(ctx);
    if (!ctx || !a || !b || !out || field < 0 || field > 1 || op < 0 || op > 2) return OG_E_INVALID;
    if (n == 0) return OG_OK;
    OG_SLOT(ctx, da, uint8_t, S_IO_A, 32 * n);
    OG_SLOT(ctx, db, uint8_t, S_IO_B, 32 * n);
    OG_SLOT(ctx, dout, uint8_t, S_IO_C, 32 * n);
    OG_TRY(clear_flag(ctx));
    H2D(ctx, da, a, 32 * n); H2D(ctx, db, b, 32 * n);
    unsigned grid = (unsigned)((n + 127) / 128);
    if (field == 0) OG_LAUNCH(ctx, k_field_op<Fq>, grid, 128, 0, op, da, db, n, dout, ctx->d_flag);
    else OG_LAUNCH(ctx, k_field_op<Fr>, grid, 128, 0, op, da, db, n, dout, ctx->d_flag);
    D2H(ctx, out, dout, 32 * n);
    return check_flag(ctx);
}

// ---- MiMC7 ----------------------------------------------------------------------------------------------
int32_t og_mimc7_constants(uint8_t* out, uint32_t* n_rounds) {
    if (!out || !n_rounds) return OG_E_INVALID;
    Fr c[MIMC_ROUNDS];
    mimc_constants_host(c);
    for (int i = 0; i < MIMC_ROUNDS; i++) host_store(out + 32 * i, c[i]);
    *n_rounds = MIMC_ROUNDS;
    return OG_OK;
}

int32_t og_mimc7_hash2(og_ctx* ctx, const uint8_t* left, const uint8_t* right, uint64_t n, uint8_t* out) {
    OG_ENTER(ctx);
    if (!ctx || !left || !right || !out) return OG_E_INVALID;
    if (n == 0) return OG_OK;
    OG_SLOT(ctx, da, uint8_t, S_IO_A, 32 * n);
    OG_SLOT(ctx, db, uint8_t, S_IO_B, 32 * n);
    OG_SLOT(ctx, dout, uint8_t, S_IO_C, 32 * n);
    OG_TRY(clear_flag(ctx));
    H2D(ctx, da, left, 32 * n); H2D(ctx, db, right, 32 * n);
    OG_TRY(mimc_hash2_dev(ctx, da, db, n, dout));
    D2H(ctx, out, dout, 32 * n);
    return check_flag(ctx);
}

int32_t og_mimc7_merkle_paths_dev(og_ctx* ctx, const uint8_t* d_leaves, const uint8_t* d_siblings, const uint32_t* d_path_bits,
                                  uint32_t n_paths, uint32_t depth, uint8_t* d_out_nodes) {
    OG_ENTER(ctx);
    if (!ctx || !d_leaves || !d_siblings || !d_path_bits || !d_out_nodes || depth > 32) return OG_E_INVALID;
    return mimc_merkle_paths_dev(ctx, d_leaves, d_siblings, d_path_bits, n_paths, depth, d_out_nodes);
}

int32_t og_mimc7_merkle_paths(og_ctx* ctx, const uint8_t* leaves, const uint8_t* siblings, const uint32_t* path_bits,
                              uint32_t n_paths, uint32_t depth, uint8_t* out_nodes) {
    OG_ENTER(ctx);
    if (!ctx || !leaves || !siblings || !path_bits || !out_nodes || depth > 32) return OG_E_INVALID;
    if (n_paths == 0) return OG_OK;
    size_t nl = 32ull * n_paths, ns = 32ull * n_paths * depth, no = 32ull * n_paths * (depth + 1);
    OG_SLOT(ctx, dl, uint8_t, S_IO_A, nl);
    OG_SLOT(ctx, ds, uint8_t, S_IO_B, ns);
    OG_SLOT(ctx, dbits, uint32_t, S_IO_C, 4ull * n_paths);
    OG_SLOT(ctx, dout, uint8_t, S_IO_D, no);
    OG_TRY(clear_flag(ctx));
    H2D(ctx, dl, leaves, nl);
    if (ns) H2D(ctx, ds, siblings, ns);
    H2D(ctx, dbits, path_bits, 4ull * n_paths);
    OG_TRY(mimc_merkle_paths_dev(ctx, dl, ds, dbits, n_paths, depth, dout));
    D2H(ctx, out_nodes, dout, no);
    return check_flag(ctx);
}

int32_t og_mimc7_merkle_build(og_ctx* ctx, const uint8_t* leaves, uint64_t n, uint8_t* out_levels) {
    OG_ENTER(ctx);
    if (!ctx || !leaves || !out_levels || n == 0 || (n & (n - 1)) || n > (1ull << 28)) return OG_E_INVALID;
    uint64_t total = 2 * n - 1;
    OG_SLOT(ctx, din, uint8_t, S_IO_A, 32 * n);
    OG_SLOT(ctx, lv, Fr, S_IO_B, sizeof(Fr) * total);
    OG_SLOT(ctx, dout, uint8_t, S_IO_C, 32 * total);
    OG_TRY(clear_flag(ctx));
    H2D(ctx, din, leaves, 32 * n);
    OG_TRY(mimc_to_mont_dev(ctx, din, n, lv));
    OG_TRY(mimc_tree_build_dev(ctx, lv, n));
    OG_TRY(mimc_from_mont_dev(ctx, lv, total, dout));
    D2H(ctx, out_levels, dout, 32 * total);
    return check_flag(ctx);
}

// nodes of levels 1..depth touched by appending n leaves at index `start` to a depth-`depth` sparse tree: one call, no
// host round trip per level.  Level l contributes ((start+n-1)>>l) - (start>>l) + 1 nodes, lowest index first.
int32_t og_mimc7_merkle_append(og_ctx* ctx, uint32_t depth, uint64_t start, const uint8_t* leaves, uint64_t n, const uint8_t* left_boundary,
                               const uint8_t* zeros, uint8_t* out_nodes) {
    OG_ENTER(ctx);
    if (!ctx || !leaves || !left_boundary || !zeros || !out_nodes || depth == 0 || depth > 32 || n == 0 || n > (1ull << 28)) return OG_E_INVALID;
    if (start + n > (1ull << depth)) return OG_E_INVALID;
    uint64_t total = 0;
    for (uint32_t l = 1; l <= depth; l++) total += ((start + n - 1) >> l) - (start >> l) + 1;
    Fr aux[64];
    for (uint32_t l = 0; l < depth; l++)
        if (!host_load(aux[l], left_boundary + 32 * l) || !host_load(aux[depth + l], zeros + 32 * l)) return OG_E_ENCODING;
    OG_SLOT(ctx, din, uint8_t, S_IO_A, 32 * n);
    OG_SLOT(ctx, nodes, Fr, S_IO_B, sizeof(Fr) * (n + total));
    OG_SLOT(ctx, dout, uint8_t, S_IO_C, 32 * total);
    OG_TRY(clear_flag(ctx));
    H2D(ctx, din, leaves, 32 * n);
    OG_TRY(mimc_to_mont_dev(ctx, din, n, nodes));
    OG_TRY(mimc_tree_append_dev(ctx, depth, start, n, aux, nodes));
    OG_TRY(mimc_from_mont_dev(ctx, nodes + n, total, dout));
    D2H(ctx, out_nodes, dout, 32 * total);
    return check_flag(ctx);
}

// ---- BabyJubJub (the reference's own signature scheme, babyjubjub/mod.rs) -----------------------------------
int32_t og_bjj_verify_batch(og_ctx* ctx, const uint8_t* pk_x, const uint8_t* pk_is_odd, const uint8_t* messages, const uint8_t* signatures,
                            uint32_t n, int32_t hash_kind, uint8_t* out_status) {
    OG_ENTER(ctx);
    if (!ctx || !pk_x || !pk_is_odd || !messages || !signatures || !out_status || hash_kind < 0 || hash_kind > 1) return OG_E_INVALID;
    if (n == 0) return OG_OK;
    OG_SLOT(ctx, dx, uint8_t, S_IO_A, 32ull * n);
    OG_SLOT(ctx, dodd, uint8_t, S_IO_B, n);
    OG_SLOT(ctx, dm, uint8_t, S_IO_C, 32ull * n);
    OG_SLOT(ctx, dsg, uint8_t, S_IO_D, 96ull * n);
    OG_SLOT(ctx, dout, uint8_t, S_IO_E, n);
    OG_TRY(clear_flag(ctx));
    H2D(ctx, dx, pk_x, 32ull * n); H2D(ctx, dodd, pk_is_odd, n); H2D(ctx, dm, messages, 32ull * n); H2D(ctx, dsg, signatures, 96ull * n);
    OG_TRY(bjj_verify_dev(ctx, dx, dodd, dm, dsg, n, hash_kind, dout));
    D2H(ctx, out_status, dout, n);
    return check_flag(ctx);
}

int32_t og_bjj_verify_batch_dev(og_ctx* ctx, const uint8_t* d_pk_x, const uint8_t* d_pk_is_odd, const uint8_t* d_messages,
                                const uint8_t* d_signatures, uint32_t n, int32_t hash_kind, uint8_t* d_out_status) {
    OG_ENTER(ctx);
    if (!ctx || hash_kind < 0 || hash_kind > 1 || (n && (!d_pk_x || !d_pk_is_odd || !d_messages || !d_signatures || !d_out_status))) return OG_E_INVALID;
    return bjj_verify_dev(ctx, d_pk_x, d_pk_is_odd, d_messages, d_signatures, n, hash_kind, d_out_status);
}
int32_t og_bjj_sign_batch_dev(og_ctx* ctx, const uint8_t* d_secret_keys, const uint8_t* d_randomness, const uint8_t* d_messages, uint32_t n,
                              int32_t hash_kind, uint8_t* d_out_pk_x, uint8_t* d_out_pk_is_odd, uint8_t* d_out_signatures, uint8_t* d_out_status) {
    OG_ENTER(ctx);
    if (!ctx || hash_kind < 0 || hash_kind > 1 ||
        (n && (!d_secret_keys || !d_randomness || !d_messages || !d_out_pk_x || !d_out_pk_is_odd || !d_out_signatures || !d_out_status))) return OG_E_INVALID;
    return bjj_sign_dev(ctx, d_secret_keys, d_randomness, d_messages, n, hash_kind, d_out_pk_x, d_out_pk_is_odd, d_out_signatures, d_out_status);
}
int32_t og_bjj_sign_batch(og_ctx* ctx, const uint8_t* secret_keys, const uint8_t* randomness, const uint8_t* messages, uint32_t n,
                          int32_t hash_kind, uint8_t* out_pk_x, uint8_t* out_pk_is_odd, uint8_t* out_signatures, uint8_t* out_status) {
    OG_ENTER(ctx);
    if (!ctx || !secret_keys || !randomness || !messages || !out_pk_x || !out_pk_is_odd || !out_signatures || !out_status || hash_kind < 0 || hash_kind > 1)
        return OG_E_INVALID;
    if (n == 0) return OG_OK;
    OG_SLOT(ctx, dsk, uint8_t, S_IO_A, 32ull * n);
    OG_SLOT(ctx, drn, uint8_t, S_IO_B, 32ull * n);
    OG_SLOT(ctx, dm, uint8_t, S_IO_C, 32ull * n);
    OG_SLOT(ctx, dpx, uint8_t, S_IO_D, 32ull * n);
    OG_SLOT(ctx, dodd, uint8_t, S_IO_E, n);
    OG_SLOT(ctx, dsg, uint8_t, S_IO_F, 96ull * n);
    OG_SLOT(ctx, dst, uint8_t, S_IO_G, n);
    OG_TRY(clear_flag(ctx));
    H2D(ctx, dsk, secret_keys, 32ull * n); H2D(ctx, drn, randomness, 32ull * n); H2D(ctx, dm, messages, 32ull * n);
    OG_TRY(bjj_sign_dev(ctx, dsk, drn, dm, n, hash_kind, dpx, dodd, dsg, dst));
    D2H(ctx, out_pk_x, dpx, 32ull * n); D2H(ctx, out_pk_is_odd, dodd, n); D2H(ctx, out_signatures, dsg, 96ull * n); D2H(ctx, out_status, dst, n);
    return check_flag(ctx);
}

// ---- encrypted notes (note_impl.cuh; spec oracle/notes.py) ------------------------------------------------------
int32_t og_note_public_keys(og_ctx* ctx, const uint8_t* view_keys, uint32_t n, uint8_t* out_pk_x, uint8_t* out_pk_is_odd) {
    OG_ENTER(ctx);
    if (n && (!view_keys || !out_pk_x || !out_pk_is_odd)) return OG_E_INVALID;
    if (n == 0) return OG_OK;
    OG_TRY(note_check_view_keys(ctx, view_keys, n));
    OG_SLOT(ctx, io, uint8_t, S_IO_NOTE, 65ull * n);
    uint8_t *dk = io, *dx = io + 32ull * n, *dodd = io + 64ull * n;
    OG_TRY(clear_flag(ctx));
    H2D(ctx, dk, view_keys, 32ull * n);
    OG_TRY(note_public_keys_dev(ctx, dk, n, dx, dodd));
    D2H(ctx, out_pk_x, dx, 32ull * n); D2H(ctx, out_pk_is_odd, dodd, n);
    return check_flag(ctx);
}

// One encrypt body and one scan body serve the three note kinds (NoteKind, mimc.cuh); every og_*note_encrypt* / og_*note_scan*
// entry point packs its arguments and calls one of these.  Owned labeled notes add one label per note to the inputs of an
// encryption; the owned kinds add one spend public key per view key to a scan's.
static bool note_encrypt_null(NoteKind kind, const NoteEncryptInputs& in, const uint32_t* labels, const uint8_t* records,
                              const uint8_t* commitments, const uint8_t* status) {
    return !in.pk_x || !in.pk_odd || !in.nullifiers || !in.secrets || !in.tokens || !in.amounts || !in.ephemerals ||
           (kind == NOTE_OWNED_LABELED && !labels) || !records || !commitments || !status;
}

static int32_t note_encrypt_dev_entry(og_ctx* ctx, NoteKind kind, const NoteEncryptInputs& d_in, const uint32_t* d_labels, uint64_t n,
                                      uint8_t* d_out_records, uint8_t* d_out_commitments, uint8_t* d_out_status) {
    OG_ENTER(ctx);
    if (n && note_encrypt_null(kind, d_in, d_labels, d_out_records, d_out_commitments, d_out_status)) return OG_E_INVALID;
    return note_encrypt_dev(ctx, d_in, n, d_out_records, d_out_commitments, d_out_status, kind, d_labels);
}

static int32_t note_encrypt_entry(og_ctx* ctx, NoteKind kind, const NoteEncryptInputs& in, const uint32_t* labels, uint64_t n,
                                  uint8_t* out_records, uint8_t* out_commitments, uint8_t* out_status) {
    OG_ENTER(ctx);
    if (n && note_encrypt_null(kind, in, labels, out_records, out_commitments, out_status)) return OG_E_INVALID;
    if (n == 0) return OG_OK;
    // per note: 5 x 32 B inputs, 8 B amount, 1 B parity (and a 4 B label) in; 160 B record, 32 B commitment, 1 B status out
    // (the u64s first, then the labels: aligned)
    const bool labeled = kind == NOTE_OWNED_LABELED;
    const uint64_t lb = labeled ? 4 : 0;
    OG_SLOT(ctx, io, uint8_t, S_IO_NOTE, (362 + lb) * n);
    uint64_t* da = reinterpret_cast<uint64_t*>(io);
    uint32_t* dla = reinterpret_cast<uint32_t*>(io + 8 * n);
    uint8_t *dx = io + (8 + lb) * n, *dnu = dx + 32 * n, *dse = dnu + 32 * n, *dto = dse + 32 * n, *de = dto + 32 * n;
    uint8_t *drec = de + 32 * n, *dcm = drec + 160 * n, *dodd = dcm + 32 * n, *dst = dodd + n;
    OG_TRY(clear_flag(ctx));
    H2D(ctx, da, in.amounts, 8 * n); H2D(ctx, dx, in.pk_x, 32 * n); H2D(ctx, dnu, in.nullifiers, 32 * n); H2D(ctx, dse, in.secrets, 32 * n);
    H2D(ctx, dto, in.tokens, 32 * n); H2D(ctx, de, in.ephemerals, 32 * n); H2D(ctx, dodd, in.pk_odd, n);
    if (labeled) H2D(ctx, dla, labels, 4 * n);
    OG_TRY(note_encrypt_dev(ctx, NoteEncryptInputs{dx, dodd, dnu, dse, dto, da, de}, n, drec, dcm, dst, kind, labeled ? dla : nullptr));
    D2H(ctx, out_records, drec, 160 * n); D2H(ctx, out_commitments, dcm, 32 * n); D2H(ctx, out_status, dst, n);
    return check_flag(ctx);
}

static bool note_scan_null(NoteKind kind, const uint8_t* view_keys, const uint8_t* spend_public_keys, uint32_t n_keys, const uint8_t* records,
                           const uint8_t* commitments, uint64_t n, const uint32_t* owner, const uint8_t* plaintexts) {
    return (n_keys && (!view_keys || (kind != NOTE_TRANSFER && !spend_public_keys))) || (n && (!records || !commitments || !owner || !plaintexts));
}

// The keys are host memory in every scan: the view keys are checked (note_check_view_keys), and for the owned kinds so are the
// spend public keys, one per view key, canonical (OG_E_ENCODING); then both are staged to the device.  *d_spend stays null
// for transfer notes, which have no owner check.
static int32_t note_stage_keys(og_ctx* ctx, NoteKind kind, const uint8_t* view_keys, const uint8_t* spend_public_keys, uint32_t n_keys,
                               const uint32_t** d_keys, const uint32_t** d_spend) {
    if (n_keys > 65535) { snprintf(ctx->err, sizeof(ctx->err), "at most 65535 view keys per scan"); return OG_E_INVALID; }
    OG_TRY(note_check_view_keys(ctx, view_keys, n_keys));
    OG_SLOT(ctx, dk, uint32_t, S_NOTE_KEYS, 32ull * n_keys);
    if (n_keys) H2D(ctx, dk, view_keys, 32ull * n_keys);
    *d_keys = dk;
    *d_spend = nullptr;
    if (kind == NOTE_TRANSFER) return OG_OK;
    for (uint32_t j = 0; j < n_keys; j++) {
        uint32_t v[8];
        memcpy(v, spend_public_keys + 32ull * j, 32);
        if (!Fr::canonical_lt_mod(v)) {
            snprintf(ctx->err, sizeof(ctx->err), "spend public key %u is not a canonical field element", j);
            return OG_E_ENCODING;
        }
    }
    OG_SLOT(ctx, ds, uint32_t, S_NOTE_SPEND_KEYS, 32ull * (n_keys ? n_keys : 1));
    if (n_keys) H2D(ctx, ds, spend_public_keys, 32ull * n_keys);
    *d_spend = ds;
    return OG_OK;
}

static int32_t note_scan_dev_entry(og_ctx* ctx, NoteKind kind, const uint8_t* view_keys, const uint8_t* spend_public_keys, uint32_t n_keys,
                                   const uint8_t* d_records, const uint8_t* d_commitments, uint64_t n, uint32_t* d_out_owner,
                                   uint8_t* d_out_plaintexts) {
    OG_ENTER(ctx);
    if (note_scan_null(kind, view_keys, spend_public_keys, n_keys, d_records, d_commitments, n, d_out_owner, d_out_plaintexts))
        return OG_E_INVALID;
    const uint32_t *dk, *ds;
    OG_TRY(note_stage_keys(ctx, kind, view_keys, spend_public_keys, n_keys, &dk, &ds));
    return note_scan_dev(ctx, dk, n_keys, d_records, d_commitments, n, d_out_owner, d_out_plaintexts, kind, ds);
}

static int32_t note_scan_entry(og_ctx* ctx, NoteKind kind, const uint8_t* view_keys, const uint8_t* spend_public_keys, uint32_t n_keys,
                               const uint8_t* records, const uint8_t* commitments, uint64_t n, uint32_t* out_owner, uint8_t* out_plaintexts) {
    OG_ENTER(ctx);
    if (note_scan_null(kind, view_keys, spend_public_keys, n_keys, records, commitments, n, out_owner, out_plaintexts)) return OG_E_INVALID;
    const uint32_t *dk, *ds;
    OG_TRY(note_stage_keys(ctx, kind, view_keys, spend_public_keys, n_keys, &dk, &ds));
    if (n == 0) return OG_OK;
    OG_SLOT(ctx, io, uint8_t, S_IO_NOTE, 324ull * n);          // 160 B record, 32 B commitment in; 4 B owner, 128 B plaintext out
    uint32_t* downer = reinterpret_cast<uint32_t*>(io);
    uint8_t *drec = io + 4 * n, *dcm = drec + 160 * n, *dpl = dcm + 32 * n;
    H2D(ctx, drec, records, 160 * n); H2D(ctx, dcm, commitments, 32 * n);
    OG_TRY(note_scan_dev(ctx, dk, n_keys, drec, dcm, n, downer, dpl, kind, ds));
    D2H(ctx, out_owner, downer, 4 * n); D2H(ctx, out_plaintexts, dpl, 128 * n);
    OG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return OG_OK;
}

int32_t og_note_encrypt_dev(og_ctx* ctx, const uint8_t* d_pk_x, const uint8_t* d_pk_is_odd, const uint8_t* d_nullifiers, const uint8_t* d_secrets,
                            const uint8_t* d_tokens, const uint64_t* d_amounts, const uint8_t* d_ephemerals, uint64_t n,
                            uint8_t* d_out_records, uint8_t* d_out_commitments, uint8_t* d_out_status) {
    return note_encrypt_dev_entry(ctx, NOTE_TRANSFER, {d_pk_x, d_pk_is_odd, d_nullifiers, d_secrets, d_tokens, d_amounts, d_ephemerals}, nullptr,
                                  n, d_out_records, d_out_commitments, d_out_status);
}
int32_t og_note_encrypt(og_ctx* ctx, const uint8_t* pk_x, const uint8_t* pk_is_odd, const uint8_t* nullifiers, const uint8_t* secrets,
                        const uint8_t* tokens, const uint64_t* amounts, const uint8_t* ephemerals, uint64_t n,
                        uint8_t* out_records, uint8_t* out_commitments, uint8_t* out_status) {
    return note_encrypt_entry(ctx, NOTE_TRANSFER, {pk_x, pk_is_odd, nullifiers, secrets, tokens, amounts, ephemerals}, nullptr, n, out_records,
                              out_commitments, out_status);
}
int32_t og_note_scan_dev(og_ctx* ctx, const uint8_t* view_keys, uint32_t n_keys, const uint8_t* d_records, const uint8_t* d_commitments,
                         uint64_t n, uint32_t* d_out_owner, uint8_t* d_out_plaintexts) {
    return note_scan_dev_entry(ctx, NOTE_TRANSFER, view_keys, nullptr, n_keys, d_records, d_commitments, n, d_out_owner, d_out_plaintexts);
}
int32_t og_note_scan(og_ctx* ctx, const uint8_t* view_keys, uint32_t n_keys, const uint8_t* records, const uint8_t* commitments, uint64_t n,
                     uint32_t* out_owner, uint8_t* out_plaintexts) {
    return note_scan_entry(ctx, NOTE_TRANSFER, view_keys, nullptr, n_keys, records, commitments, n, out_owner, out_plaintexts);
}

// ---- spend-key notes: encryption and scanning (NOTE_OWNED: the nullifier and secret fields carry owner and blinding) ---------
int32_t og_owned_note_encrypt_dev(og_ctx* ctx, const uint8_t* d_pk_x, const uint8_t* d_pk_is_odd, const uint8_t* d_owners,
                                  const uint8_t* d_blindings, const uint8_t* d_tokens, const uint64_t* d_amounts, const uint8_t* d_ephemerals,
                                  uint64_t n, uint8_t* d_out_records, uint8_t* d_out_commitments, uint8_t* d_out_status) {
    return note_encrypt_dev_entry(ctx, NOTE_OWNED, {d_pk_x, d_pk_is_odd, d_owners, d_blindings, d_tokens, d_amounts, d_ephemerals}, nullptr, n,
                                  d_out_records, d_out_commitments, d_out_status);
}
int32_t og_owned_note_encrypt(og_ctx* ctx, const uint8_t* pk_x, const uint8_t* pk_is_odd, const uint8_t* owners, const uint8_t* blindings,
                              const uint8_t* tokens, const uint64_t* amounts, const uint8_t* ephemerals, uint64_t n,
                              uint8_t* out_records, uint8_t* out_commitments, uint8_t* out_status) {
    return note_encrypt_entry(ctx, NOTE_OWNED, {pk_x, pk_is_odd, owners, blindings, tokens, amounts, ephemerals}, nullptr, n, out_records,
                              out_commitments, out_status);
}
int32_t og_owned_note_scan_dev(og_ctx* ctx, const uint8_t* view_keys, const uint8_t* spend_public_keys, uint32_t n_keys,
                               const uint8_t* d_records, const uint8_t* d_commitments, uint64_t n, uint32_t* d_out_owner,
                               uint8_t* d_out_plaintexts) {
    return note_scan_dev_entry(ctx, NOTE_OWNED, view_keys, spend_public_keys, n_keys, d_records, d_commitments, n, d_out_owner,
                               d_out_plaintexts);
}
int32_t og_owned_note_scan(og_ctx* ctx, const uint8_t* view_keys, const uint8_t* spend_public_keys, uint32_t n_keys, const uint8_t* records,
                           const uint8_t* commitments, uint64_t n, uint32_t* out_owner, uint8_t* out_plaintexts) {
    return note_scan_entry(ctx, NOTE_OWNED, view_keys, spend_public_keys, n_keys, records, commitments, n, out_owner, out_plaintexts);
}

// ---- owned labeled notes: encryption and scanning (NOTE_OWNED_LABELED) --------------------------------------------------
int32_t og_owned_labeled_note_encrypt_dev(og_ctx* ctx, const uint8_t* d_pk_x, const uint8_t* d_pk_is_odd, const uint8_t* d_owners,
                                          const uint8_t* d_blindings, const uint8_t* d_tokens, const uint64_t* d_amounts,
                                          const uint32_t* d_labels, const uint8_t* d_ephemerals, uint64_t n, uint8_t* d_out_records,
                                          uint8_t* d_out_commitments, uint8_t* d_out_status) {
    return note_encrypt_dev_entry(ctx, NOTE_OWNED_LABELED, {d_pk_x, d_pk_is_odd, d_owners, d_blindings, d_tokens, d_amounts, d_ephemerals},
                                  d_labels, n, d_out_records, d_out_commitments, d_out_status);
}
int32_t og_owned_labeled_note_encrypt(og_ctx* ctx, const uint8_t* pk_x, const uint8_t* pk_is_odd, const uint8_t* owners,
                                      const uint8_t* blindings, const uint8_t* tokens, const uint64_t* amounts, const uint32_t* labels,
                                      const uint8_t* ephemerals, uint64_t n, uint8_t* out_records, uint8_t* out_commitments,
                                      uint8_t* out_status) {
    return note_encrypt_entry(ctx, NOTE_OWNED_LABELED, {pk_x, pk_is_odd, owners, blindings, tokens, amounts, ephemerals}, labels, n,
                              out_records, out_commitments, out_status);
}
int32_t og_owned_labeled_note_scan_dev(og_ctx* ctx, const uint8_t* view_keys, const uint8_t* spend_public_keys, uint32_t n_keys,
                                       const uint8_t* d_records, const uint8_t* d_commitments, uint64_t n, uint32_t* d_out_owner,
                                       uint8_t* d_out_plaintexts) {
    return note_scan_dev_entry(ctx, NOTE_OWNED_LABELED, view_keys, spend_public_keys, n_keys, d_records, d_commitments, n, d_out_owner,
                               d_out_plaintexts);
}
int32_t og_owned_labeled_note_scan(og_ctx* ctx, const uint8_t* view_keys, const uint8_t* spend_public_keys, uint32_t n_keys,
                                   const uint8_t* records, const uint8_t* commitments, uint64_t n, uint32_t* out_owner,
                                   uint8_t* out_plaintexts) {
    return note_scan_entry(ctx, NOTE_OWNED_LABELED, view_keys, spend_public_keys, n_keys, records, commitments, n, out_owner, out_plaintexts);
}

// ---- MSM --------------------------------------------------------------------------------------------------
}  // extern "C"

// one body for the G1 and the G2 entry point of each pair: F = Fq (64-byte points) or Fq2 (128-byte points)
template <class F>
static int32_t msm_entry_dev(og_ctx* ctx, const uint8_t* d_points, const uint8_t* d_scalars, uint64_t n, uint8_t* d_out) {
    OG_ENTER(ctx);
    if (!ctx || !d_out || (n && (!d_points || !d_scalars))) return OG_E_INVALID;
    return msm_dev<F>(ctx, d_points, d_scalars, n, d_out);
}
template <class F>
static int32_t msm_entry(og_ctx* ctx, const uint8_t* points, const uint8_t* scalars, uint64_t n, uint8_t* out) {
    constexpr size_t PB = sizeof(Affine<F>);
    OG_ENTER(ctx);
    if (!ctx || !out || (n && (!points || !scalars))) return OG_E_INVALID;
    OG_SLOT(ctx, dp, uint8_t, S_IO_A, PB * n);
    OG_SLOT(ctx, ds, uint8_t, S_IO_B, 32 * n);
    OG_SLOT(ctx, dout, uint8_t, S_IO_C, PB);
    OG_TRY(clear_flag(ctx));
    if (n) { H2D(ctx, dp, points, PB * n); H2D(ctx, ds, scalars, 32 * n); }
    OG_TRY(msm_dev<F>(ctx, dp, ds, n, dout));
    D2H(ctx, out, dout, PB);
    return check_flag(ctx);
}
template <class F>
static int32_t sum_entry(og_ctx* ctx, const uint8_t* points, uint64_t n, uint8_t* out) {
    constexpr size_t PB = sizeof(Affine<F>);
    OG_ENTER(ctx);
    if (!ctx || !out || (n && !points)) return OG_E_INVALID;
    OG_SLOT(ctx, dp, uint8_t, S_IO_A, PB * n);
    OG_SLOT(ctx, dout, uint8_t, S_IO_C, PB);
    OG_TRY(clear_flag(ctx));
    if (n) H2D(ctx, dp, points, PB * n);
    OG_TRY(sum_dev<F>(ctx, dp, n, dout));
    D2H(ctx, out, dout, PB);
    return check_flag(ctx);
}
template <class F>
static int32_t sum_entry_dev(og_ctx* ctx, const uint8_t* d_points, uint64_t n, uint8_t* d_out) {
    OG_ENTER(ctx);
    if (!d_out || (n && !d_points)) return OG_E_INVALID;
    return sum_dev<F>(ctx, d_points, n, d_out);
}
template <class F>
static int32_t generator_mul_entry_dev(og_ctx* ctx, const uint8_t* d_scalars, uint64_t n, uint8_t* d_out_points) {
    OG_ENTER(ctx);
    if (n && (!d_scalars || !d_out_points)) return OG_E_INVALID;
    if (n == 0) return OG_OK;
    OG_SLOT(ctx, dp, Affine<F>, S_IO_B, sizeof(Affine<F>) * n);
    OG_TRY(fixed_base_mul(ctx, d_scalars, n, dp));
    return points_mont_to_bytes(ctx, dp, n, d_out_points);
}
// out[i] = scalars[i] * G (fixed-base, generator of G1 / G2): used by the setup and to synthesise MSM inputs
template <class F>
static int32_t generator_mul_entry(og_ctx* ctx, const uint8_t* scalars, uint64_t n, uint8_t* out_points) {
    constexpr size_t PB = sizeof(Affine<F>);
    OG_ENTER(ctx);
    if (!ctx || (n && (!scalars || !out_points))) return OG_E_INVALID;
    if (n == 0) return OG_OK;
    OG_SLOT(ctx, ds, uint8_t, S_IO_A, 32 * n);
    OG_SLOT(ctx, dp, Affine<F>, S_IO_B, PB * n);
    OG_SLOT(ctx, dout, uint8_t, S_IO_C, PB * n);
    OG_TRY(clear_flag(ctx));
    H2D(ctx, ds, scalars, 32 * n);
    OG_TRY(fixed_base_mul(ctx, ds, n, dp));
    OG_TRY(points_mont_to_bytes(ctx, dp, n, dout));
    D2H(ctx, out_points, dout, PB * n);
    return check_flag(ctx);
}

extern "C" {

int32_t og_msm_g1_dev(og_ctx* ctx, const uint8_t* d_points, const uint8_t* d_scalars, uint64_t n, uint8_t* d_out64) { return msm_entry_dev<Fq>(ctx, d_points, d_scalars, n, d_out64); }
int32_t og_msm_g2_dev(og_ctx* ctx, const uint8_t* d_points, const uint8_t* d_scalars, uint64_t n, uint8_t* d_out128) { return msm_entry_dev<Fq2>(ctx, d_points, d_scalars, n, d_out128); }
int32_t og_msm_g1(og_ctx* ctx, const uint8_t* points, const uint8_t* scalars, uint64_t n, uint8_t* out64) { return msm_entry<Fq>(ctx, points, scalars, n, out64); }
int32_t og_msm_g2(og_ctx* ctx, const uint8_t* points, const uint8_t* scalars, uint64_t n, uint8_t* out128) { return msm_entry<Fq2>(ctx, points, scalars, n, out128); }
int32_t og_g1_sum(og_ctx* ctx, const uint8_t* points, uint64_t n, uint8_t* out64) { return sum_entry<Fq>(ctx, points, n, out64); }
int32_t og_g2_sum(og_ctx* ctx, const uint8_t* points, uint64_t n, uint8_t* out128) { return sum_entry<Fq2>(ctx, points, n, out128); }
int32_t og_g1_sum_dev(og_ctx* ctx, const uint8_t* d_points, uint64_t n, uint8_t* d_out64) { return sum_entry_dev<Fq>(ctx, d_points, n, d_out64); }
int32_t og_g2_sum_dev(og_ctx* ctx, const uint8_t* d_points, uint64_t n, uint8_t* d_out128) { return sum_entry_dev<Fq2>(ctx, d_points, n, d_out128); }
int32_t og_g1_generator_mul_dev(og_ctx* ctx, const uint8_t* d_scalars, uint64_t n, uint8_t* d_out_points) { return generator_mul_entry_dev<Fq>(ctx, d_scalars, n, d_out_points); }
int32_t og_g2_generator_mul_dev(og_ctx* ctx, const uint8_t* d_scalars, uint64_t n, uint8_t* d_out_points) { return generator_mul_entry_dev<Fq2>(ctx, d_scalars, n, d_out_points); }
int32_t og_g1_generator_mul(og_ctx* ctx, const uint8_t* scalars, uint64_t n, uint8_t* out_points) { return generator_mul_entry<Fq>(ctx, scalars, n, out_points); }
int32_t og_g2_generator_mul(og_ctx* ctx, const uint8_t* scalars, uint64_t n, uint8_t* out_points) { return generator_mul_entry<Fq2>(ctx, scalars, n, out_points); }

// ---- NTT ----------------------------------------------------------------------------------------------------
int32_t og_ntt_dev(og_ctx* ctx, uint8_t* d_data, uint32_t log_n, uint32_t batch, int32_t inverse, int32_t coset) {
    OG_ENTER(ctx);
    if (!ctx || !d_data || log_n > 27 || !aligned32(d_data)) return OG_E_INVALID;
    uint64_t tot = (uint64_t)batch << log_n;
    if (tot == 0) return OG_OK;
    OG_SLOT(ctx, work, Fr, S_NTT_DATA, sizeof(Fr) * tot * 2);
    OG_TRY(mimc_to_mont_dev(ctx, d_data, tot, work));
    OG_TRY(ntt_mont_dev(ctx, work, work + tot, log_n, batch, inverse, coset));
    return mimc_from_mont_dev(ctx, work, tot, d_data);
}
int32_t og_ntt(og_ctx* ctx, uint8_t* data, uint32_t log_n, uint32_t batch, int32_t inverse, int32_t coset) {
    OG_ENTER(ctx);
    if (!ctx || !data || log_n > 27) return OG_E_INVALID;
    uint64_t tot = (uint64_t)batch << log_n;
    if (tot == 0) return OG_OK;
    OG_SLOT(ctx, dd, uint8_t, S_IO_A, 32 * tot);
    OG_TRY(clear_flag(ctx));
    H2D(ctx, dd, data, 32 * tot);
    OG_TRY(og_ntt_dev(ctx, dd, log_n, batch, inverse, coset));
    D2H(ctx, data, dd, 32 * tot);
    return check_flag(ctx);
}

// ---- the statements (the statement table, mimc.cuh) -----------------------------------------------------------------
// Every og_<statement>_* entry point packs its input arrays, in C ABI order, into a StatementInputs and calls one of these.
// Checks run in one order for every statement: ctx, null pointers, key on this device, key of this statement, batch 0.
static bool depth_ok(Statement s, uint32_t depth) { return STATEMENTS[s].takes_depth ? depth >= 1 && depth <= 32 : depth == 0; }

static bool any_null(Statement s, const StatementInputs& in) {
    for (uint32_t k = 0; k < STATEMENTS[s].n_inputs; k++) if (!in.p[k]) return true;
    return false;
}

static int32_t statement_r1cs_info(Statement s, uint32_t depth, uint32_t* n_constraints, uint32_t* n_vars, uint32_t* n_pub,
                                   uint32_t* log_m) {
    if (!depth_ok(s, depth)) return OG_E_INVALID;
    const StatementShape sh = STATEMENTS[s].shape(depth);
    const uint32_t np = STATEMENTS[s].n_pub;
    if (n_constraints) *n_constraints = sh.n_constraints;
    if (n_vars) *n_vars = sh.n_vars;
    if (n_pub) *n_pub = np;
    if (log_m) *log_m = groth16_domain_log(sh.n_constraints, np);
    return OG_OK;
}

static int32_t statement_r1cs_export(Statement s, uint32_t depth, int32_t which, uint32_t* row_ptr, uint32_t* col_idx, uint8_t* coeffs,
                                     uint64_t* nnz) {
    if (!depth_ok(s, depth) || which < 0 || which > 2 || !nnz) return OG_E_INVALID;
    R1cs cs = statement_r1cs(s, depth);
    const Csr& M = which == 0 ? cs.A : (which == 1 ? cs.B : cs.C);
    *nnz = M.col.size();
    if (!row_ptr || !col_idx || !coeffs) return OG_OK;
    memcpy(row_ptr, M.row_ptr.data(), 4 * M.row_ptr.size());
    memcpy(col_idx, M.col.data(), 4 * M.col.size());
    for (size_t i = 0; i < M.val.size(); i++) host_store(coeffs + 32 * i, M.val[i]);
    return OG_OK;
}

// the host input arrays of a batch, copied into one device slot (each array 256-byte aligned)
static int32_t stage_statement_inputs(og_ctx* ctx, Statement s, uint32_t depth, uint32_t batch, const StatementInputs& h,
                                      StatementInputs& d) {
    const StatementDesc& S = STATEMENTS[s];
    uint64_t off[STATEMENT_MAX_INPUTS], tot = 0;
    for (uint32_t k = 0; k < S.n_inputs; k++) { off[k] = tot; tot += (S.input_bytes(k, depth) * batch + 255) & ~255ull; }
    OG_SLOT(ctx, base, uint8_t, S_IO_STATEMENT, tot);
    for (uint32_t k = 0; k < S.n_inputs; k++) {
        H2D(ctx, base + off[k], h.p[k], S.input_bytes(k, depth) * batch);
        d.p[k] = base + off[k];
    }
    return OG_OK;
}

static int32_t statement_witness(og_ctx* ctx, Statement s, uint32_t depth, const StatementInputs& in, uint32_t batch, uint8_t* witnesses) {
    OG_ENTER(ctx);
    if (!depth_ok(s, depth) || any_null(s, in) || !witnesses) return OG_E_INVALID;
    if (batch == 0) return OG_OK;
    const uint64_t out_bytes = 32ull * batch * STATEMENTS[s].shape(depth).n_vars;
    StatementInputs d;
    OG_TRY(stage_statement_inputs(ctx, s, depth, batch, in, d));
    OG_SLOT(ctx, dout, uint8_t, S_IO_F, out_bytes);
    OG_TRY(clear_flag(ctx));
    OG_TRY(statement_witness_bytes_dev(ctx, s, depth, d, batch, dout));
    D2H(ctx, witnesses, dout, out_bytes);
    return check_flag(ctx);
}

static int32_t statement_prove(og_ctx* ctx, const og_pk* pk, Statement s, const StatementInputs& in, uint32_t batch, const uint8_t* rs,
                               uint8_t* proofs, uint8_t* public_out) {
    OG_ENTER(ctx);
    if (!pk || any_null(s, in) || !rs || !proofs) return OG_E_INVALID;
    OG_PK_CHECK(ctx, pk);
    const int32_t depth = statement_key_depth(pk, s);
    if (depth < 0) return OG_E_INVALID;
    if (batch == 0) return OG_OK;
    uint32_t n_pub; pk_info(pk, nullptr, &n_pub, nullptr, nullptr);
    StatementInputs d;
    OG_TRY(stage_statement_inputs(ctx, s, (uint32_t)depth, batch, in, d));
    OG_SLOT(ctx, drs, uint8_t, S_IO_F, 64ull * batch);
    OG_SLOT(ctx, dpr, uint8_t, S_IO_G, 256ull * batch);
    OG_SLOT(ctx, dpub, uint8_t, S_IO_H, 32ull * batch * n_pub);
    OG_TRY(clear_flag(ctx));
    H2D(ctx, drs, rs, 64ull * batch);
    OG_TRY(prove_statement_dev(ctx, pk, s, d, batch, drs, dpr, public_out ? dpub : nullptr));
    D2H(ctx, proofs, dpr, 256ull * batch);
    if (public_out) D2H(ctx, public_out, dpub, 32ull * batch * n_pub);
    return check_flag(ctx);
}

static int32_t statement_prove_dev(og_ctx* ctx, const og_pk* pk, Statement s, const StatementInputs& d_in, uint32_t batch,
                                   const uint8_t* d_rs, uint8_t* d_proofs, uint8_t* d_public_out) {
    OG_ENTER(ctx);
    if (!pk || any_null(s, d_in) || !d_rs || !d_proofs) return OG_E_INVALID;
    OG_PK_CHECK(ctx, pk);
    return prove_statement_dev(ctx, pk, s, d_in, batch, d_rs, d_proofs, d_public_out);
}

// ---- the note hashes (the note-hash table, mimc.cuh) ------------------------------------------------------------------
// Every og_* note hash packs its columns, in C ABI order, into a StatementInputs and calls this.  Column k is staged in slot
// S_IO_A + k and the output in the slot after the last column.
static int32_t note_hash_entry(og_ctx* ctx, NoteHash h, const StatementInputs& cols, uint64_t n, uint8_t* out) {
    OG_ENTER(ctx);
    const NoteHashDesc& H = NOTE_HASHES[h];
    for (uint32_t k = 0; k < H.n_cols; k++) if (!cols.p[k]) return OG_E_INVALID;
    if (!out) return OG_E_INVALID;
    if (n == 0) return OG_OK;
    uint8_t* d[NOTE_HASH_MAX_COLUMNS];
    for (uint32_t k = 0; k < H.n_cols; k++) {
        OG_SLOT(ctx, dk, uint8_t, S_IO_A + k, H.cols[k] * n);
        d[k] = dk;
    }
    OG_SLOT(ctx, dout, uint8_t, S_IO_A + H.n_cols, 32 * n);
    OG_TRY(clear_flag(ctx));
    StatementInputs dc;
    for (uint32_t k = 0; k < H.n_cols; k++) {
        H2D(ctx, d[k], cols.p[k], H.cols[k] * n);
        dc.p[k] = d[k];
    }
    OG_TRY(note_hash_dev(ctx, h, dc, n, dout));
    D2H(ctx, out, dout, 32 * n);
    return check_flag(ctx);
}

// ---- withdraw statement ----------------------------------------------------------------------------------------
int32_t og_withdraw_r1cs_info(uint32_t depth, uint32_t* n_constraints, uint32_t* n_vars, uint32_t* n_pub, uint32_t* log_m) {
    return statement_r1cs_info(ST_WITHDRAW, depth, n_constraints, n_vars, n_pub, log_m);
}
int32_t og_withdraw_r1cs_export(uint32_t depth, int32_t which, uint32_t* row_ptr, uint32_t* col_idx, uint8_t* coeffs, uint64_t* nnz) {
    return statement_r1cs_export(ST_WITHDRAW, depth, which, row_ptr, col_idx, coeffs, nnz);
}
int32_t og_withdraw_witness(og_ctx* ctx, uint32_t depth, const uint8_t* nullifiers, const uint8_t* secrets, const uint8_t* recipients,
                            const uint8_t* siblings, const uint32_t* path_bits, uint32_t batch, uint8_t* witnesses) {
    return statement_witness(ctx, ST_WITHDRAW, depth, {nullifiers, secrets, recipients, siblings, path_bits}, batch, witnesses);
}

// ---- deposit statement ----------------------------------------------------------------------------------------
int32_t og_deposit_r1cs_info(uint32_t* n_constraints, uint32_t* n_vars, uint32_t* n_pub, uint32_t* log_m) {
    return statement_r1cs_info(ST_DEPOSIT, 0, n_constraints, n_vars, n_pub, log_m);
}
int32_t og_deposit_r1cs_export(int32_t which, uint32_t* row_ptr, uint32_t* col_idx, uint8_t* coeffs, uint64_t* nnz) {
    return statement_r1cs_export(ST_DEPOSIT, 0, which, row_ptr, col_idx, coeffs, nnz);
}
int32_t og_deposit_witness(og_ctx* ctx, const uint8_t* nullifiers, const uint8_t* secrets, const uint8_t* depositors, uint32_t batch,
                           uint8_t* witnesses) {
    return statement_witness(ctx, ST_DEPOSIT, 0, {nullifiers, secrets, depositors}, batch, witnesses);
}

// ---- transfer statement ---------------------------------------------------------------------------------------
int32_t og_transfer_r1cs_info(uint32_t depth, uint32_t* n_constraints, uint32_t* n_vars, uint32_t* n_pub, uint32_t* log_m) {
    return statement_r1cs_info(ST_TRANSFER, depth, n_constraints, n_vars, n_pub, log_m);
}
int32_t og_transfer_r1cs_export(uint32_t depth, int32_t which, uint32_t* row_ptr, uint32_t* col_idx, uint8_t* coeffs, uint64_t* nnz) {
    return statement_r1cs_export(ST_TRANSFER, depth, which, row_ptr, col_idx, coeffs, nnz);
}
int32_t og_transfer_witness(og_ctx* ctx, uint32_t depth, const uint8_t* roots, const uint8_t* tokens, const uint8_t* recipients,
                            const uint8_t* in_nullifiers, const uint8_t* in_secrets, const uint64_t* in_amounts,
                            const uint8_t* in_siblings, const uint32_t* in_path_bits,
                            const uint8_t* out_nullifiers, const uint8_t* out_secrets, const uint64_t* out_amounts,
                            uint32_t batch, uint8_t* witnesses) {
    return statement_witness(ctx, ST_TRANSFER, depth, {roots, tokens, recipients, in_nullifiers, in_secrets, in_amounts, in_siblings,
                                                       in_path_bits, out_nullifiers, out_secrets, out_amounts}, batch, witnesses);
}

// ---- association-set withdraw statement ---------------------------------------------------------------------------
int32_t og_association_r1cs_info(uint32_t depth, uint32_t* n_constraints, uint32_t* n_vars, uint32_t* n_pub, uint32_t* log_m) {
    return statement_r1cs_info(ST_ASSOCIATION, depth, n_constraints, n_vars, n_pub, log_m);
}
int32_t og_association_r1cs_export(uint32_t depth, int32_t which, uint32_t* row_ptr, uint32_t* col_idx, uint8_t* coeffs, uint64_t* nnz) {
    return statement_r1cs_export(ST_ASSOCIATION, depth, which, row_ptr, col_idx, coeffs, nnz);
}
int32_t og_association_witness(og_ctx* ctx, uint32_t depth, const uint8_t* nullifiers, const uint8_t* secrets, const uint8_t* recipients,
                               const uint8_t* siblings, const uint32_t* path_bits, const uint8_t* assoc_siblings,
                               const uint32_t* assoc_path_bits, uint32_t batch, uint8_t* witnesses) {
    return statement_witness(ctx, ST_ASSOCIATION, depth, {nullifiers, secrets, recipients, siblings, path_bits, assoc_siblings,
                                                          assoc_path_bits}, batch, witnesses);
}

// ---- exclusion withdraw statement ----------------------------------------------------------------------------------
int32_t og_exclusion_r1cs_info(uint32_t depth, uint32_t* n_constraints, uint32_t* n_vars, uint32_t* n_pub, uint32_t* log_m) {
    return statement_r1cs_info(ST_EXCLUSION, depth, n_constraints, n_vars, n_pub, log_m);
}
int32_t og_exclusion_r1cs_export(uint32_t depth, int32_t which, uint32_t* row_ptr, uint32_t* col_idx, uint8_t* coeffs, uint64_t* nnz) {
    return statement_r1cs_export(ST_EXCLUSION, depth, which, row_ptr, col_idx, coeffs, nnz);
}
int32_t og_exclusion_witness(og_ctx* ctx, uint32_t depth, const uint8_t* nullifiers, const uint8_t* secrets, const uint8_t* recipients,
                             const uint8_t* siblings, const uint32_t* path_bits, const uint64_t* excl_low, const uint64_t* excl_next,
                             const uint8_t* excl_siblings, const uint32_t* excl_path_bits, uint32_t batch, uint8_t* witnesses) {
    return statement_witness(ctx, ST_EXCLUSION, depth, {nullifiers, secrets, recipients, siblings, path_bits, excl_low, excl_next,
                                                        excl_siblings, excl_path_bits}, batch, witnesses);
}

// ---- labeled notes and the labeled withdraw statement --------------------------------------------------------------
int32_t og_labeled_precommitments(og_ctx* ctx, const uint8_t* nullifiers, const uint8_t* secrets, uint64_t n, uint8_t* out) {
    return note_hash_entry(ctx, NH_LABELED_PRECOMMITMENTS, {nullifiers, secrets}, n, out);
}
int32_t og_labeled_leaves(og_ctx* ctx, const uint8_t* precommitments, const uint8_t* tokens, const uint64_t* amounts, const uint32_t* labels,
                          uint64_t n, uint8_t* out) {
    return note_hash_entry(ctx, NH_LABELED_LEAVES, {precommitments, tokens, amounts, labels}, n, out);
}
int32_t og_labeled_r1cs_info(uint32_t depth, uint32_t* n_constraints, uint32_t* n_vars, uint32_t* n_pub, uint32_t* log_m) {
    return statement_r1cs_info(ST_LABELED, depth, n_constraints, n_vars, n_pub, log_m);
}
int32_t og_labeled_r1cs_export(uint32_t depth, int32_t which, uint32_t* row_ptr, uint32_t* col_idx, uint8_t* coeffs, uint64_t* nnz) {
    return statement_r1cs_export(ST_LABELED, depth, which, row_ptr, col_idx, coeffs, nnz);
}
int32_t og_labeled_witness(og_ctx* ctx, uint32_t depth, const uint8_t* tokens, const uint8_t* recipients, const uint64_t* withdrawn,
                           const uint8_t* nullifiers, const uint8_t* secrets, const uint64_t* amounts, const uint32_t* labels,
                           const uint8_t* siblings, const uint32_t* path_bits, const uint8_t* change_nullifiers, const uint8_t* change_secrets,
                           const uint64_t* excl_low, const uint64_t* excl_next, const uint8_t* excl_siblings, const uint32_t* excl_path_bits,
                           uint32_t batch, uint8_t* witnesses) {
    return statement_witness(ctx, ST_LABELED, depth, {tokens, recipients, withdrawn, nullifiers, secrets, amounts, labels, siblings, path_bits,
                                                      change_nullifiers, change_secrets, excl_low, excl_next, excl_siblings, excl_path_bits},
                             batch, witnesses);
}

// ---- labeled association withdraw statement -------------------------------------------------------------------------
int32_t og_labeled_association_r1cs_info(uint32_t depth, uint32_t* n_constraints, uint32_t* n_vars, uint32_t* n_pub, uint32_t* log_m) {
    return statement_r1cs_info(ST_LABELED_ASSOCIATION, depth, n_constraints, n_vars, n_pub, log_m);
}
int32_t og_labeled_association_r1cs_export(uint32_t depth, int32_t which, uint32_t* row_ptr, uint32_t* col_idx, uint8_t* coeffs,
                                           uint64_t* nnz) {
    return statement_r1cs_export(ST_LABELED_ASSOCIATION, depth, which, row_ptr, col_idx, coeffs, nnz);
}
int32_t og_labeled_association_witness(og_ctx* ctx, uint32_t depth, const uint8_t* tokens, const uint8_t* recipients,
                                       const uint64_t* withdrawn, const uint8_t* nullifiers, const uint8_t* secrets,
                                       const uint64_t* amounts, const uint32_t* labels, const uint8_t* siblings, const uint32_t* path_bits,
                                       const uint8_t* change_nullifiers, const uint8_t* change_secrets, const uint8_t* assoc_siblings,
                                       const uint32_t* assoc_path_bits, uint32_t batch, uint8_t* witnesses) {
    return statement_witness(ctx, ST_LABELED_ASSOCIATION, depth, {tokens, recipients, withdrawn, nullifiers, secrets, amounts, labels,
                                                                  siblings, path_bits, change_nullifiers, change_secrets, assoc_siblings,
                                                                  assoc_path_bits}, batch, witnesses);
}

// ---- spend-key notes and the owned transfer statement ---------------------------------------------------------------
int32_t og_owned_public_keys(og_ctx* ctx, const uint8_t* spend_keys, uint64_t n, uint8_t* out) {
    return note_hash_entry(ctx, NH_OWNED_PUBLIC_KEYS, {spend_keys}, n, out);
}
int32_t og_owned_commitments(og_ctx* ctx, const uint8_t* owners, const uint8_t* blindings, const uint8_t* tokens, const uint64_t* amounts,
                             uint64_t n, uint8_t* out) {
    return note_hash_entry(ctx, NH_OWNED_COMMITMENTS, {owners, blindings, tokens, amounts}, n, out);
}
int32_t og_owned_nullifiers(og_ctx* ctx, const uint8_t* spend_keys, const uint8_t* commitments, const uint32_t* indices, uint64_t n,
                            uint8_t* out) {
    return note_hash_entry(ctx, NH_OWNED_NULLIFIERS, {spend_keys, commitments, indices}, n, out);
}
int32_t og_owned_transfer_r1cs_info(uint32_t depth, uint32_t* n_constraints, uint32_t* n_vars, uint32_t* n_pub, uint32_t* log_m) {
    return statement_r1cs_info(ST_OWNED_TRANSFER, depth, n_constraints, n_vars, n_pub, log_m);
}
int32_t og_owned_transfer_r1cs_export(uint32_t depth, int32_t which, uint32_t* row_ptr, uint32_t* col_idx, uint8_t* coeffs, uint64_t* nnz) {
    return statement_r1cs_export(ST_OWNED_TRANSFER, depth, which, row_ptr, col_idx, coeffs, nnz);
}
int32_t og_owned_transfer_witness(og_ctx* ctx, uint32_t depth, const uint8_t* roots, const uint8_t* tokens, const uint8_t* recipients,
                                  const uint8_t* in_spend_keys, const uint8_t* in_blindings, const uint64_t* in_amounts,
                                  const uint8_t* in_siblings, const uint32_t* in_path_bits,
                                  const uint8_t* out_owners, const uint8_t* out_blindings, const uint64_t* out_amounts,
                                  uint32_t batch, uint8_t* witnesses) {
    return statement_witness(ctx, ST_OWNED_TRANSFER, depth, {roots, tokens, recipients, in_spend_keys, in_blindings, in_amounts, in_siblings,
                                                             in_path_bits, out_owners, out_blindings, out_amounts}, batch, witnesses);
}

// ---- owned labeled notes and the owned labeled transfer statement ----------------------------------------------------
int32_t og_owned_labeled_precommitments(og_ctx* ctx, const uint8_t* owners, const uint8_t* blindings, uint64_t n, uint8_t* out) {
    return note_hash_entry(ctx, NH_OWNED_LABELED_PRECOMMITMENTS, {owners, blindings}, n, out);
}
int32_t og_owned_labeled_leaves(og_ctx* ctx, const uint8_t* precommitments, const uint8_t* tokens, const uint64_t* amounts,
                                const uint32_t* labels, uint64_t n, uint8_t* out) {
    return note_hash_entry(ctx, NH_OWNED_LABELED_LEAVES, {precommitments, tokens, amounts, labels}, n, out);
}
int32_t og_owned_labeled_transfer_r1cs_info(uint32_t depth, uint32_t* n_constraints, uint32_t* n_vars, uint32_t* n_pub, uint32_t* log_m) {
    return statement_r1cs_info(ST_OWNED_LABELED_TRANSFER, depth, n_constraints, n_vars, n_pub, log_m);
}
int32_t og_owned_labeled_transfer_r1cs_export(uint32_t depth, int32_t which, uint32_t* row_ptr, uint32_t* col_idx, uint8_t* coeffs,
                                              uint64_t* nnz) {
    return statement_r1cs_export(ST_OWNED_LABELED_TRANSFER, depth, which, row_ptr, col_idx, coeffs, nnz);
}
int32_t og_owned_labeled_transfer_witness(og_ctx* ctx, uint32_t depth, const uint8_t* roots, const uint8_t* tokens, const uint8_t* recipients,
                                          const uint64_t* withdrawn, const uint32_t* labels, const uint8_t* in_spend_keys,
                                          const uint8_t* in_blindings, const uint64_t* in_amounts, const uint8_t* in_siblings,
                                          const uint32_t* in_path_bits, const uint8_t* out_owners, const uint8_t* out_blindings,
                                          const uint64_t* out_amounts, const uint8_t* assoc_siblings, const uint32_t* assoc_path_bits,
                                          uint32_t batch, uint8_t* witnesses) {
    return statement_witness(ctx, ST_OWNED_LABELED_TRANSFER, depth, {roots, tokens, recipients, withdrawn, labels, in_spend_keys, in_blindings,
                                                                     in_amounts, in_siblings, in_path_bits, out_owners, out_blindings,
                                                                     out_amounts, assoc_siblings, assoc_path_bits}, batch, witnesses);
}

// ---- the ragequit statement --------------------------------------------------------------------------------------
int32_t og_ragequit_r1cs_info(uint32_t depth, uint32_t* n_constraints, uint32_t* n_vars, uint32_t* n_pub, uint32_t* log_m) {
    return statement_r1cs_info(ST_RAGEQUIT, depth, n_constraints, n_vars, n_pub, log_m);
}
int32_t og_ragequit_r1cs_export(uint32_t depth, int32_t which, uint32_t* row_ptr, uint32_t* col_idx, uint8_t* coeffs, uint64_t* nnz) {
    return statement_r1cs_export(ST_RAGEQUIT, depth, which, row_ptr, col_idx, coeffs, nnz);
}
int32_t og_ragequit_witness(og_ctx* ctx, uint32_t depth, const uint8_t* roots, const uint8_t* tokens, const uint8_t* recipients,
                            const uint64_t* amounts, const uint32_t* labels, const uint8_t* spend_keys, const uint8_t* blindings,
                            const uint8_t* siblings, const uint32_t* path_bits, uint32_t batch, uint8_t* witnesses) {
    return statement_witness(ctx, ST_RAGEQUIT, depth, {roots, tokens, recipients, amounts, labels, spend_keys, blindings, siblings, path_bits},
                             batch, witnesses);
}

// ---- Groth16 -------------------------------------------------------------------------------------------------------
int32_t og_groth16_setup(og_ctx* ctx, uint32_t n_constraints, uint32_t n_vars, uint32_t n_pub,
                         const uint32_t* a_row_ptr, const uint32_t* a_col, const uint8_t* a_coeffs,
                         const uint32_t* b_row_ptr, const uint32_t* b_col, const uint8_t* b_coeffs,
                         const uint32_t* c_row_ptr, const uint32_t* c_col, const uint8_t* c_coeffs,
                         const uint8_t* toxic160, uint8_t* pk_out, uint64_t* pk_len, uint8_t* vk_out, uint64_t* vk_len) {
    OG_ENTER(ctx);
    if (!ctx || !pk_len || !vk_len || ((pk_out || vk_out) && !toxic160)) return OG_E_INVALID;
    const uint32_t* row_ptr[3] = {a_row_ptr, b_row_ptr, c_row_ptr};
    const uint32_t* col[3] = {a_col, b_col, c_col};
    const uint8_t* coeffs[3] = {a_coeffs, b_coeffs, c_coeffs};
    try {
        return setup_generic(ctx, n_constraints, n_vars, n_pub, row_ptr, col, coeffs, toxic160, pk_out, pk_len, vk_out, vk_len);
    } catch (const std::bad_alloc&) {           // a shape whose host-side QAP evaluation does not fit in memory
        snprintf(ctx->err, sizeof(ctx->err), "setup: host allocation failed");
        return OG_E_NOMEM;
    }
}
int32_t og_groth16_setup_withdraw(og_ctx* ctx, uint32_t depth, const uint8_t* toxic160, uint8_t* pk_out, uint64_t* pk_len,
                                  uint8_t* vk_out, uint64_t* vk_len) {
    OG_ENTER(ctx);
    if (!ctx || !pk_len || !vk_len || ((pk_out || vk_out) && !toxic160)) return OG_E_INVALID;
    return setup_withdraw(ctx, depth, toxic160, pk_out, pk_len, vk_out, vk_len);
}
int32_t og_load_pk(og_ctx* ctx, const uint8_t* pk_bytes, uint64_t len, og_pk** out) {
    OG_ENTER(ctx);
    if (!ctx || !pk_bytes || !out) return OG_E_INVALID;
    return pk_load(ctx, pk_bytes, len, out);
}
void og_free_pk(og_pk* pk) { pk_free(pk); }
int32_t og_pk_info(const og_pk* pk, uint32_t* n_vars, uint32_t* n_pub, uint32_t* log_m, uint32_t* depth) {
    if (!pk) return OG_E_INVALID;
    pk_info(pk, n_vars, n_pub, log_m, depth);
    return OG_OK;
}

int32_t og_pk_window_bits(const og_pk* pk, uint32_t* c3) {
    if (!pk || !c3) return OG_E_INVALID;
    pk_window_bits(pk, c3);
    return OG_OK;
}

int32_t og_groth16_prove(og_ctx* ctx, const og_pk* pk, const uint8_t* witnesses, uint32_t batch, const uint8_t* rs, uint8_t* proofs) {
    OG_ENTER(ctx);
    if (!ctx || !pk || !witnesses || !rs || !proofs) return OG_E_INVALID;
    OG_PK_CHECK(ctx, pk);
    if (batch == 0) return OG_OK;
    uint32_t nv; pk_info(pk, &nv, nullptr, nullptr, nullptr);
    OG_SLOT(ctx, dw, uint8_t, S_IO_A, 32ull * batch * nv);
    OG_SLOT(ctx, drs, uint8_t, S_IO_B, 64ull * batch);
    OG_SLOT(ctx, dpr, uint8_t, S_IO_C, 256ull * batch);
    OG_TRY(clear_flag(ctx));
    H2D(ctx, dw, witnesses, 32ull * batch * nv); H2D(ctx, drs, rs, 64ull * batch);
    OG_TRY(prove_witness_dev(ctx, pk, dw, batch, drs, dpr));
    D2H(ctx, proofs, dpr, 256ull * batch);
    return check_flag(ctx);
}

int32_t og_groth16_prove_withdraw_dev(og_ctx* ctx, const og_pk* pk, const uint8_t* d_nullifiers, const uint8_t* d_secrets,
                                      const uint8_t* d_recipients, const uint8_t* d_siblings, const uint32_t* d_path_bits, uint32_t batch,
                                      const uint8_t* d_rs, uint8_t* d_proofs, uint8_t* d_public_out) {
    return statement_prove_dev(ctx, pk, ST_WITHDRAW, {d_nullifiers, d_secrets, d_recipients, d_siblings, d_path_bits}, batch, d_rs,
                               d_proofs, d_public_out);
}

int32_t og_groth16_prove_withdraw(og_ctx* ctx, const og_pk* pk, const uint8_t* nullifiers, const uint8_t* secrets, const uint8_t* recipients,
                                  const uint8_t* siblings, const uint32_t* path_bits, uint32_t batch, const uint8_t* rs, uint8_t* proofs,
                                  uint8_t* public_out) {
    return statement_prove(ctx, pk, ST_WITHDRAW, {nullifiers, secrets, recipients, siblings, path_bits}, batch, rs, proofs, public_out);
}

int32_t og_groth16_prove_deposit_dev(og_ctx* ctx, const og_pk* pk, const uint8_t* d_nullifiers, const uint8_t* d_secrets,
                                     const uint8_t* d_depositors, uint32_t batch, const uint8_t* d_rs, uint8_t* d_proofs,
                                     uint8_t* d_public_out) {
    return statement_prove_dev(ctx, pk, ST_DEPOSIT, {d_nullifiers, d_secrets, d_depositors}, batch, d_rs, d_proofs, d_public_out);
}

int32_t og_groth16_prove_deposit(og_ctx* ctx, const og_pk* pk, const uint8_t* nullifiers, const uint8_t* secrets, const uint8_t* depositors,
                                 uint32_t batch, const uint8_t* rs, uint8_t* proofs, uint8_t* public_out) {
    return statement_prove(ctx, pk, ST_DEPOSIT, {nullifiers, secrets, depositors}, batch, rs, proofs, public_out);
}

int32_t og_groth16_prove_transfer_dev(og_ctx* ctx, const og_pk* pk, const uint8_t* d_roots, const uint8_t* d_tokens,
                                      const uint8_t* d_recipients, const uint8_t* d_in_nullifiers, const uint8_t* d_in_secrets,
                                      const uint64_t* d_in_amounts, const uint8_t* d_in_siblings, const uint32_t* d_in_path_bits,
                                      const uint8_t* d_out_nullifiers, const uint8_t* d_out_secrets, const uint64_t* d_out_amounts,
                                      uint32_t batch, const uint8_t* d_rs, uint8_t* d_proofs, uint8_t* d_public_out) {
    return statement_prove_dev(ctx, pk, ST_TRANSFER, {d_roots, d_tokens, d_recipients, d_in_nullifiers, d_in_secrets, d_in_amounts,
                                                      d_in_siblings, d_in_path_bits, d_out_nullifiers, d_out_secrets, d_out_amounts},
                               batch, d_rs, d_proofs, d_public_out);
}

int32_t og_groth16_prove_transfer(og_ctx* ctx, const og_pk* pk, const uint8_t* roots, const uint8_t* tokens, const uint8_t* recipients,
                                  const uint8_t* in_nullifiers, const uint8_t* in_secrets, const uint64_t* in_amounts,
                                  const uint8_t* in_siblings, const uint32_t* in_path_bits,
                                  const uint8_t* out_nullifiers, const uint8_t* out_secrets, const uint64_t* out_amounts,
                                  uint32_t batch, const uint8_t* rs, uint8_t* proofs, uint8_t* public_out) {
    return statement_prove(ctx, pk, ST_TRANSFER, {roots, tokens, recipients, in_nullifiers, in_secrets, in_amounts, in_siblings,
                                                  in_path_bits, out_nullifiers, out_secrets, out_amounts}, batch, rs, proofs, public_out);
}

int32_t og_groth16_prove_association_dev(og_ctx* ctx, const og_pk* pk, const uint8_t* d_nullifiers, const uint8_t* d_secrets,
                                         const uint8_t* d_recipients, const uint8_t* d_siblings, const uint32_t* d_path_bits,
                                         const uint8_t* d_assoc_siblings, const uint32_t* d_assoc_path_bits, uint32_t batch,
                                         const uint8_t* d_rs, uint8_t* d_proofs, uint8_t* d_public_out) {
    return statement_prove_dev(ctx, pk, ST_ASSOCIATION, {d_nullifiers, d_secrets, d_recipients, d_siblings, d_path_bits, d_assoc_siblings,
                                                         d_assoc_path_bits}, batch, d_rs, d_proofs, d_public_out);
}

int32_t og_groth16_prove_association(og_ctx* ctx, const og_pk* pk, const uint8_t* nullifiers, const uint8_t* secrets,
                                     const uint8_t* recipients, const uint8_t* siblings, const uint32_t* path_bits,
                                     const uint8_t* assoc_siblings, const uint32_t* assoc_path_bits, uint32_t batch, const uint8_t* rs,
                                     uint8_t* proofs, uint8_t* public_out) {
    return statement_prove(ctx, pk, ST_ASSOCIATION, {nullifiers, secrets, recipients, siblings, path_bits, assoc_siblings, assoc_path_bits},
                           batch, rs, proofs, public_out);
}

int32_t og_groth16_prove_exclusion_dev(og_ctx* ctx, const og_pk* pk, const uint8_t* d_nullifiers, const uint8_t* d_secrets,
                                       const uint8_t* d_recipients, const uint8_t* d_siblings, const uint32_t* d_path_bits,
                                       const uint64_t* d_excl_low, const uint64_t* d_excl_next, const uint8_t* d_excl_siblings,
                                       const uint32_t* d_excl_path_bits, uint32_t batch, const uint8_t* d_rs, uint8_t* d_proofs,
                                       uint8_t* d_public_out) {
    return statement_prove_dev(ctx, pk, ST_EXCLUSION, {d_nullifiers, d_secrets, d_recipients, d_siblings, d_path_bits, d_excl_low,
                                                       d_excl_next, d_excl_siblings, d_excl_path_bits}, batch, d_rs, d_proofs, d_public_out);
}

int32_t og_groth16_prove_exclusion(og_ctx* ctx, const og_pk* pk, const uint8_t* nullifiers, const uint8_t* secrets,
                                   const uint8_t* recipients, const uint8_t* siblings, const uint32_t* path_bits, const uint64_t* excl_low,
                                   const uint64_t* excl_next, const uint8_t* excl_siblings, const uint32_t* excl_path_bits, uint32_t batch,
                                   const uint8_t* rs, uint8_t* proofs, uint8_t* public_out) {
    return statement_prove(ctx, pk, ST_EXCLUSION, {nullifiers, secrets, recipients, siblings, path_bits, excl_low, excl_next, excl_siblings,
                                                   excl_path_bits}, batch, rs, proofs, public_out);
}

int32_t og_groth16_prove_labeled_dev(og_ctx* ctx, const og_pk* pk, const uint8_t* d_tokens, const uint8_t* d_recipients,
                                     const uint64_t* d_withdrawn, const uint8_t* d_nullifiers, const uint8_t* d_secrets, const uint64_t* d_amounts,
                                     const uint32_t* d_labels, const uint8_t* d_siblings, const uint32_t* d_path_bits,
                                     const uint8_t* d_change_nullifiers, const uint8_t* d_change_secrets, const uint64_t* d_excl_low,
                                     const uint64_t* d_excl_next, const uint8_t* d_excl_siblings, const uint32_t* d_excl_path_bits, uint32_t batch,
                                     const uint8_t* d_rs, uint8_t* d_proofs, uint8_t* d_public_out) {
    return statement_prove_dev(ctx, pk, ST_LABELED, {d_tokens, d_recipients, d_withdrawn, d_nullifiers, d_secrets, d_amounts, d_labels, d_siblings,
                                                     d_path_bits, d_change_nullifiers, d_change_secrets, d_excl_low, d_excl_next, d_excl_siblings,
                                                     d_excl_path_bits}, batch, d_rs, d_proofs, d_public_out);
}

int32_t og_groth16_prove_labeled(og_ctx* ctx, const og_pk* pk, const uint8_t* tokens, const uint8_t* recipients, const uint64_t* withdrawn,
                                 const uint8_t* nullifiers, const uint8_t* secrets, const uint64_t* amounts, const uint32_t* labels,
                                 const uint8_t* siblings, const uint32_t* path_bits, const uint8_t* change_nullifiers,
                                 const uint8_t* change_secrets, const uint64_t* excl_low, const uint64_t* excl_next, const uint8_t* excl_siblings,
                                 const uint32_t* excl_path_bits, uint32_t batch, const uint8_t* rs, uint8_t* proofs, uint8_t* public_out) {
    return statement_prove(ctx, pk, ST_LABELED, {tokens, recipients, withdrawn, nullifiers, secrets, amounts, labels, siblings, path_bits,
                                                 change_nullifiers, change_secrets, excl_low, excl_next, excl_siblings, excl_path_bits},
                           batch, rs, proofs, public_out);
}

int32_t og_groth16_prove_labeled_association_dev(og_ctx* ctx, const og_pk* pk, const uint8_t* d_tokens, const uint8_t* d_recipients,
                                                 const uint64_t* d_withdrawn, const uint8_t* d_nullifiers, const uint8_t* d_secrets,
                                                 const uint64_t* d_amounts, const uint32_t* d_labels, const uint8_t* d_siblings,
                                                 const uint32_t* d_path_bits, const uint8_t* d_change_nullifiers,
                                                 const uint8_t* d_change_secrets, const uint8_t* d_assoc_siblings,
                                                 const uint32_t* d_assoc_path_bits, uint32_t batch, const uint8_t* d_rs,
                                                 uint8_t* d_proofs, uint8_t* d_public_out) {
    return statement_prove_dev(ctx, pk, ST_LABELED_ASSOCIATION, {d_tokens, d_recipients, d_withdrawn, d_nullifiers, d_secrets, d_amounts,
                                                                 d_labels, d_siblings, d_path_bits, d_change_nullifiers, d_change_secrets,
                                                                 d_assoc_siblings, d_assoc_path_bits}, batch, d_rs, d_proofs, d_public_out);
}

int32_t og_groth16_prove_labeled_association(og_ctx* ctx, const og_pk* pk, const uint8_t* tokens, const uint8_t* recipients,
                                             const uint64_t* withdrawn, const uint8_t* nullifiers, const uint8_t* secrets,
                                             const uint64_t* amounts, const uint32_t* labels, const uint8_t* siblings,
                                             const uint32_t* path_bits, const uint8_t* change_nullifiers, const uint8_t* change_secrets,
                                             const uint8_t* assoc_siblings, const uint32_t* assoc_path_bits, uint32_t batch,
                                             const uint8_t* rs, uint8_t* proofs, uint8_t* public_out) {
    return statement_prove(ctx, pk, ST_LABELED_ASSOCIATION, {tokens, recipients, withdrawn, nullifiers, secrets, amounts, labels, siblings,
                                                             path_bits, change_nullifiers, change_secrets, assoc_siblings, assoc_path_bits},
                           batch, rs, proofs, public_out);
}

int32_t og_groth16_prove_owned_transfer_dev(og_ctx* ctx, const og_pk* pk, const uint8_t* d_roots, const uint8_t* d_tokens,
                                            const uint8_t* d_recipients, const uint8_t* d_in_spend_keys, const uint8_t* d_in_blindings,
                                            const uint64_t* d_in_amounts, const uint8_t* d_in_siblings, const uint32_t* d_in_path_bits,
                                            const uint8_t* d_out_owners, const uint8_t* d_out_blindings, const uint64_t* d_out_amounts,
                                            uint32_t batch, const uint8_t* d_rs, uint8_t* d_proofs, uint8_t* d_public_out) {
    return statement_prove_dev(ctx, pk, ST_OWNED_TRANSFER, {d_roots, d_tokens, d_recipients, d_in_spend_keys, d_in_blindings, d_in_amounts,
                                                            d_in_siblings, d_in_path_bits, d_out_owners, d_out_blindings, d_out_amounts},
                               batch, d_rs, d_proofs, d_public_out);
}

int32_t og_groth16_prove_owned_transfer(og_ctx* ctx, const og_pk* pk, const uint8_t* roots, const uint8_t* tokens, const uint8_t* recipients,
                                        const uint8_t* in_spend_keys, const uint8_t* in_blindings, const uint64_t* in_amounts,
                                        const uint8_t* in_siblings, const uint32_t* in_path_bits,
                                        const uint8_t* out_owners, const uint8_t* out_blindings, const uint64_t* out_amounts,
                                        uint32_t batch, const uint8_t* rs, uint8_t* proofs, uint8_t* public_out) {
    return statement_prove(ctx, pk, ST_OWNED_TRANSFER, {roots, tokens, recipients, in_spend_keys, in_blindings, in_amounts, in_siblings,
                                                        in_path_bits, out_owners, out_blindings, out_amounts}, batch, rs, proofs, public_out);
}

int32_t og_groth16_prove_owned_labeled_transfer_dev(og_ctx* ctx, const og_pk* pk, const uint8_t* d_roots, const uint8_t* d_tokens,
                                                    const uint8_t* d_recipients, const uint64_t* d_withdrawn, const uint32_t* d_labels,
                                                    const uint8_t* d_in_spend_keys, const uint8_t* d_in_blindings, const uint64_t* d_in_amounts,
                                                    const uint8_t* d_in_siblings, const uint32_t* d_in_path_bits, const uint8_t* d_out_owners,
                                                    const uint8_t* d_out_blindings, const uint64_t* d_out_amounts,
                                                    const uint8_t* d_assoc_siblings, const uint32_t* d_assoc_path_bits, uint32_t batch,
                                                    const uint8_t* d_rs, uint8_t* d_proofs, uint8_t* d_public_out) {
    return statement_prove_dev(ctx, pk, ST_OWNED_LABELED_TRANSFER, {d_roots, d_tokens, d_recipients, d_withdrawn, d_labels, d_in_spend_keys,
                                                                    d_in_blindings, d_in_amounts, d_in_siblings, d_in_path_bits, d_out_owners,
                                                                    d_out_blindings, d_out_amounts, d_assoc_siblings, d_assoc_path_bits},
                               batch, d_rs, d_proofs, d_public_out);
}

int32_t og_groth16_prove_owned_labeled_transfer(og_ctx* ctx, const og_pk* pk, const uint8_t* roots, const uint8_t* tokens,
                                                const uint8_t* recipients, const uint64_t* withdrawn, const uint32_t* labels,
                                                const uint8_t* in_spend_keys, const uint8_t* in_blindings, const uint64_t* in_amounts,
                                                const uint8_t* in_siblings, const uint32_t* in_path_bits, const uint8_t* out_owners,
                                                const uint8_t* out_blindings, const uint64_t* out_amounts, const uint8_t* assoc_siblings,
                                                const uint32_t* assoc_path_bits, uint32_t batch, const uint8_t* rs, uint8_t* proofs,
                                                uint8_t* public_out) {
    return statement_prove(ctx, pk, ST_OWNED_LABELED_TRANSFER, {roots, tokens, recipients, withdrawn, labels, in_spend_keys, in_blindings,
                                                                in_amounts, in_siblings, in_path_bits, out_owners, out_blindings, out_amounts,
                                                                assoc_siblings, assoc_path_bits}, batch, rs, proofs, public_out);
}

int32_t og_groth16_prove_ragequit_dev(og_ctx* ctx, const og_pk* pk, const uint8_t* d_roots, const uint8_t* d_tokens, const uint8_t* d_recipients,
                                      const uint64_t* d_amounts, const uint32_t* d_labels, const uint8_t* d_spend_keys,
                                      const uint8_t* d_blindings, const uint8_t* d_siblings, const uint32_t* d_path_bits, uint32_t batch,
                                      const uint8_t* d_rs, uint8_t* d_proofs, uint8_t* d_public_out) {
    return statement_prove_dev(ctx, pk, ST_RAGEQUIT, {d_roots, d_tokens, d_recipients, d_amounts, d_labels, d_spend_keys, d_blindings,
                                                      d_siblings, d_path_bits}, batch, d_rs, d_proofs, d_public_out);
}

int32_t og_groth16_prove_ragequit(og_ctx* ctx, const og_pk* pk, const uint8_t* roots, const uint8_t* tokens, const uint8_t* recipients,
                                  const uint64_t* amounts, const uint32_t* labels, const uint8_t* spend_keys, const uint8_t* blindings,
                                  const uint8_t* siblings, const uint32_t* path_bits, uint32_t batch, const uint8_t* rs, uint8_t* proofs,
                                  uint8_t* public_out) {
    return statement_prove(ctx, pk, ST_RAGEQUIT, {roots, tokens, recipients, amounts, labels, spend_keys, blindings, siblings, path_bits},
                           batch, rs, proofs, public_out);
}

int32_t og_pk_prover_plan(const og_pk* pk, uint32_t batch, uint32_t* chunk, uint32_t* lanes, uint64_t* scratch_bytes_per_lane) {
    if (!pk) return OG_E_INVALID;
    pk_prover_plan(pk, batch, chunk, lanes, scratch_bytes_per_lane);
    return OG_OK;
}

int32_t og_groth16_h_evals(og_ctx* ctx, const og_pk* pk, const uint8_t* witness, uint8_t* out) {
    OG_ENTER(ctx);
    if (!ctx || !pk || !witness || !out) return OG_E_INVALID;
    OG_PK_CHECK(ctx, pk);
    uint32_t nv, log_m; pk_info(pk, &nv, nullptr, &log_m, nullptr);
    OG_SLOT(ctx, dw, uint8_t, S_IO_A, 32ull * nv);
    OG_SLOT(ctx, dout, uint8_t, S_IO_B, 32ull << log_m);
    OG_TRY(clear_flag(ctx));
    H2D(ctx, dw, witness, 32ull * nv);
    OG_TRY(h_evals_dev(ctx, pk, dw, dout));
    D2H(ctx, out, dout, 32ull << log_m);
    return check_flag(ctx);
}

int32_t og_groth16_verify(const uint8_t* vk, uint64_t vk_len, const uint8_t* public_inputs, uint32_t n_pub, const uint8_t* proof256) {
    if (!vk || !proof256 || (n_pub && !public_inputs)) return OG_E_INVALID;
    return groth16_verify_host(vk, vk_len, public_inputs, n_pub, proof256);
}

// ---- setup ceremony (ceremony.cu) -------------------------------------------------------------------------------------
int32_t og_ptau_new(og_ctx* ctx, uint32_t log_max, uint8_t* out, uint64_t* out_len) {
    OG_ENTER(ctx);
    return ptau_new(ctx, log_max, out, out_len);
}
int32_t og_ptau_contribute(og_ctx* ctx, const uint8_t* acc, uint64_t acc_len, const uint8_t* secrets96, const uint8_t* nonces96,
                           uint8_t* acc_out, uint64_t* acc_out_len, uint8_t* record_out, uint64_t* record_len) {
    OG_ENTER(ctx);
    return ptau_contribute(ctx, acc, acc_len, secrets96, nonces96, acc_out, acc_out_len, record_out, record_len);
}
int32_t og_ptau_verify(og_ctx* ctx, const uint8_t* prev, uint64_t prev_len, const uint8_t* next, uint64_t next_len, const uint8_t* record,
                       uint64_t record_len) {
    OG_ENTER(ctx);
    return ptau_verify(ctx, prev, prev_len, next, next_len, record, record_len);
}
int32_t og_ptau_prepare(og_ctx* ctx, const uint8_t* acc, uint64_t acc_len, uint32_t n_constraints, uint32_t n_vars, uint32_t n_pub,
                        const uint32_t* a_row_ptr, const uint32_t* a_col, const uint8_t* a_coeffs,
                        const uint32_t* b_row_ptr, const uint32_t* b_col, const uint8_t* b_coeffs,
                        const uint32_t* c_row_ptr, const uint32_t* c_col, const uint8_t* c_coeffs,
                        uint8_t* pk_out, uint64_t* pk_len, uint8_t* vk_out, uint64_t* vk_len) {
    OG_ENTER(ctx);
    if (!pk_len || !vk_len) return OG_E_INVALID;
    const uint32_t* row_ptr[3] = {a_row_ptr, b_row_ptr, c_row_ptr};
    const uint32_t* col[3] = {a_col, b_col, c_col};
    const uint8_t* coeffs[3] = {a_coeffs, b_coeffs, c_coeffs};
    try {
        R1cs cs;
        OG_TRY(load_r1cs(n_constraints, n_vars, n_pub, row_ptr, col, coeffs, cs));
        return ptau_prepare(ctx, acc, acc_len, cs, 0, pk_out, pk_len, vk_out, vk_len);
    } catch (const std::bad_alloc&) {
        snprintf(ctx->err, sizeof(ctx->err), "ptau_prepare: host allocation failed");
        return OG_E_NOMEM;
    }
}
int32_t og_ptau_prepare_withdraw(og_ctx* ctx, const uint8_t* acc, uint64_t acc_len, uint32_t depth, uint8_t* pk_out, uint64_t* pk_len,
                                 uint8_t* vk_out, uint64_t* vk_len) {
    OG_ENTER(ctx);
    if (depth == 0 || depth > 32 || !pk_len || !vk_len) return OG_E_INVALID;
    return ptau_prepare(ctx, acc, acc_len, WithdrawBuilder::build(depth), depth, pk_out, pk_len, vk_out, vk_len);
}
int32_t og_phase2_contribute(og_ctx* ctx, const uint8_t* pk, uint64_t pk_len, const uint8_t* vk, uint64_t vk_len, const uint8_t* delta32,
                             const uint8_t* nonce32, uint8_t* pk_out, uint64_t* pk_out_len, uint8_t* vk_out, uint64_t* vk_out_len,
                             uint8_t* record_out, uint64_t* record_len) {
    OG_ENTER(ctx);
    return phase2_contribute(ctx, pk, pk_len, vk, vk_len, delta32, nonce32, pk_out, pk_out_len, vk_out, vk_out_len, record_out, record_len);
}
int32_t og_phase2_verify(og_ctx* ctx, const uint8_t* pk_prev, uint64_t pk_prev_len, const uint8_t* vk_prev, uint64_t vk_prev_len,
                         const uint8_t* pk_next, uint64_t pk_next_len, const uint8_t* vk_next, uint64_t vk_next_len, const uint8_t* record,
                         uint64_t record_len) {
    OG_ENTER(ctx);
    return phase2_verify(ctx, pk_prev, pk_prev_len, vk_prev, vk_prev_len, pk_next, pk_next_len, vk_next, vk_next_len, record, record_len);
}
int32_t og_scale_points(og_ctx* ctx, int32_t g2, const uint8_t* points, const uint8_t* scalars, uint64_t n, int32_t per_point, uint8_t* out) {
    OG_ENTER(ctx);
    if (g2 < 0 || g2 > 1 || (n && (!points || !scalars || !out))) return OG_E_INVALID;
    if (n == 0) return OG_OK;
    const uint64_t pb = g2 ? 128 : 64, ns = per_point ? n : 1;
    OG_SLOT(ctx, dp, uint8_t, S_IO_A, pb * n);
    OG_SLOT(ctx, ds, uint8_t, S_IO_B, 32 * ns);
    OG_TRY(clear_flag(ctx));
    H2D(ctx, dp, points, pb * n); H2D(ctx, ds, scalars, 32 * ns);
    OG_TRY(scale_points_dev(ctx, g2, dp, ds, n, per_point, dp));
    D2H(ctx, out, dp, pb * n);
    return check_flag(ctx);
}
int32_t og_intt_points(og_ctx* ctx, int32_t g2, uint8_t* points, uint32_t log_m) {
    OG_ENTER(ctx);
    if (g2 < 0 || g2 > 1 || !points || log_m > 25) return OG_E_INVALID;
    const uint64_t pb = (g2 ? 128ull : 64ull) << log_m;
    OG_SLOT(ctx, dp, uint8_t, S_IO_A, pb);
    OG_TRY(clear_flag(ctx));
    H2D(ctx, dp, points, pb);
    OG_TRY(intt_points_dev(ctx, g2, dp, log_m));
    D2H(ctx, points, dp, pb);
    return check_flag(ctx);
}

// ---- test/debug probes of the MSM units (msm.cu) ----------------------------------------------------------------------
// Every argument is checked before anything is staged or launched: msm_buckets trusts its lists and its heavy plan.  The cap and the
// segment length follow n_entries_max / n_keys (msm.cuh: msm_heavy_cap / msm_heavy_seg); n_entries_max < 2^30 keeps them and the
// segment arithmetic of k_heavy_plan / k_bucket_heavy within 32 bits, and the segment count is checked against the d_lvl scratch the
// segment sums are written into (which an n_entries_max below sum(counts), or avg >= 512, can exceed).
int32_t og_msm_bucket_sums(og_ctx* ctx, int32_t g2, const uint8_t* points, uint32_t n_points, const uint32_t* counts,
                           const uint32_t* entries, uint32_t n_groups, uint32_t nb, uint64_t n_entries_max, int32_t few_groups,
                           uint8_t* out_totals, uint8_t* out_buckets) {
    OG_ENTER(ctx);
    if (g2 < 0 || g2 > 1 || !counts || !out_totals || (n_points && !points)) return OG_E_INVALID;
    if (nb < 2 || nb > 32768 || (nb & (nb - 1)) || n_groups == 0 || n_groups > 65535 || (uint64_t)n_groups * nb > (1u << 26)) {
        snprintf(ctx->err, sizeof(ctx->err), "nb must be a power of two in [2, 2^15], n_groups in [1, 65535], n_groups * nb <= 2^26");
        return OG_E_INVALID;
    }
    const uint32_t n_keys = n_groups * nb;
    std::vector<uint32_t> offsets;
    try { offsets.resize((size_t)n_keys + 1); } catch (const std::bad_alloc&) { return OG_E_NOMEM; }
    uint64_t total = 0;
    for (uint32_t k = 0; k < n_keys; k++) {
        offsets[k] = (uint32_t)total;
        total += counts[k];
        if (total > 0xFFFFFFFFull) { snprintf(ctx->err, sizeof(ctx->err), "sum(counts) does not fit 32 bits"); return OG_E_INVALID; }
    }
    offsets[n_keys] = (uint32_t)total;
    if (n_entries_max < total || n_entries_max >= (1ull << 30)) {
        snprintf(ctx->err, sizeof(ctx->err), "n_entries_max must lie in [sum(counts), 2^30)");
        return OG_E_INVALID;
    }
    const uint64_t avg = n_entries_max / n_keys;
    const uint32_t cap = msm_heavy_cap(avg), seg = msm_heavy_seg(avg);
    uint64_t n_seg = 0;
    for (uint32_t k = 0; k < n_keys; k++)
        if (counts[k] > cap) n_seg += (counts[k] + (uint64_t)seg - 1) / seg;
    if (n_seg > msm_lvl_elems(n_groups, nb)) {
        snprintf(ctx->err, sizeof(ctx->err), "%llu heavy segments exceed the %llu segment sums of the level scratch", (unsigned long long)n_seg,
                 (unsigned long long)msm_lvl_elems(n_groups, nb));
        return OG_E_INVALID;
    }
    if (total && !entries) return OG_E_INVALID;
    for (uint64_t i = 0; i < total; i++)
        if ((entries[i] >> 1) >= n_points) { snprintf(ctx->err, sizeof(ctx->err), "entry %llu: point index out of range", (unsigned long long)i); return OG_E_INVALID; }
    const uint64_t pb = g2 ? 128 : 64;
    OG_SLOT(ctx, dp, uint8_t, S_IO_A, pb * n_points);
    OG_SLOT(ctx, de, uint32_t, S_IO_B, 4 * total);
    OG_SLOT(ctx, dc, uint32_t, S_IO_C, 4ull * n_keys);
    OG_SLOT(ctx, doff, uint32_t, S_IO_D, 4ull * (n_keys + 1ull));
    OG_SLOT(ctx, dtot, uint8_t, S_IO_E, pb * n_groups);
    uint8_t* dbk = nullptr;
    if (out_buckets) { dbk = (uint8_t*)ctx->slot(S_IO_F, pb * n_keys); if (!dbk) return OG_E_NOMEM; }
    OG_TRY(clear_flag(ctx));
    if (n_points) H2D(ctx, dp, points, pb * n_points);
    if (total) H2D(ctx, de, entries, 4 * total);
    H2D(ctx, dc, counts, 4ull * n_keys);
    H2D(ctx, doff, offsets.data(), 4ull * (n_keys + 1ull));
    if (g2) OG_TRY(msm_bucket_sums<Fq2>(ctx, dp, n_points, de, doff, dc, n_groups, nb, n_entries_max, few_groups != 0, dtot, dbk));
    else OG_TRY(msm_bucket_sums<Fq>(ctx, dp, n_points, de, doff, dc, n_groups, nb, n_entries_max, few_groups != 0, dtot, dbk));
    D2H(ctx, out_totals, dtot, pb * n_groups);
    if (out_buckets) D2H(ctx, out_buckets, dbk, pb * n_keys);
    return check_flag(ctx);
}

int32_t og_field_probe_raw(og_ctx* ctx, int32_t unit, int32_t op, const uint8_t* a, const uint8_t* b, uint64_t n, uint8_t* out) {
    OG_ENTER(ctx);
    const bool op_ok = unit ? (op >= 0 && op <= 7) : ((op >= 0 && op <= 3) || (op >= 8 && op <= 14));   // G1: 4-7 unused
    if (unit < 0 || unit > 1 || !op_ok || (n && (!a || !b || !out))) return OG_E_INVALID;
    if (n == 0) return OG_OK;
    const uint64_t eb = unit ? 64 : 32;
    OG_SLOT(ctx, da, uint8_t, S_IO_A, eb * n);
    OG_SLOT(ctx, db, uint8_t, S_IO_B, eb * n);
    OG_SLOT(ctx, dout, uint8_t, S_IO_C, eb * n);
    H2D(ctx, da, a, eb * n); H2D(ctx, db, b, eb * n);
    if (unit) OG_TRY(field_probe_raw<Fq2>(ctx, op, da, db, n, dout));
    else OG_TRY(field_probe_raw<Fq>(ctx, op, da, db, n, dout));
    D2H(ctx, out, dout, eb * n);
    OG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return OG_OK;
}

}  // extern "C"
