// owshen_b200/csrc/msm.cu -- bucket-method (Pippenger) multi-scalar multiplication on BN254 G1/G2
// for sm_90a.  BASELINE configs 3 and 5 and the inner engine of the batched Groth16 prover.
//
// No counterpart in the reference (SURVEY.md section 0).  Pipeline (DESIGN.md section 5.3):
//   1. k_digits<false>   signed c-bit digits of every scalar, histogram of (group, bucket) keys
//   2. k_scan            exclusive prefix sum of the histogram
//   3. k_digits<true>    counting-sort scatter of (point index, sign) entries  -> coalesced bucket lists
//      (the batched prover sorts with a two-pass partitioned counting sort instead: k_sort_part_count, k_sort_part_scatter,
//      k_sort_local)
//   4. k_bucket_acc      one thread per bucket: XYZZ += affine point (8M+2S), accumulator in registers
//      k_bucket_heavy    buckets above a cap get a whole CTA (witness-like scalars: 0/1 pile-ups)
//   5. k_reduce_level    sum_b (b+1) B_b by 32-way running sums, log_32(nb) levels
//   6. k_group_total / k_horner
// All arithmetic is 8x32-bit Montgomery limbs in registers (fp.cuh); the kernels are bound by the
// integer multiply-add pipe, not HBM: a G1 mixed add moves 64 B + 4 B and costs ~3.5k instructions.
#include "msm.cuh"
#include "glv.cuh"
#include <stdlib.h>
// Compiled twice: -DOG_MSM_G1 (G1 instantiations + the curve-independent sort) and -DOG_MSM_G2.
#if !defined(OG_MSM_G1) && !defined(OG_MSM_G2)
#error "compile msm.cu with -DOG_MSM_G1 or -DOG_MSM_G2"
#endif

namespace og {

// ---- boundary conversions ---------------------------------------------------------------------------
template <class F> struct FieldIO;
template <> struct FieldIO<Fq> {
    static constexpr int BYTES = 32;
    static __device__ __forceinline__ Fq load(const uint8_t* p, int* flag) { return load_canonical<Fq>(p, flag); }
    static __device__ __forceinline__ void store(uint8_t* p, const Fq& v) { store_canonical(p, v); }
};
template <> struct FieldIO<Fq2> {
    static constexpr int BYTES = 64;
    static __device__ __forceinline__ Fq2 load(const uint8_t* p, int* flag) {
        return Fq2{load_canonical<Fq>(p, flag), load_canonical<Fq>(p + 32, flag)};
    }
    static __device__ __forceinline__ void store(uint8_t* p, const Fq2& v) { store_canonical(p, v.c0); store_canonical(p + 32, v.c1); }
};

template <class F>
__global__ void __launch_bounds__(128) k_points_to_mont(const uint8_t* __restrict__ in, uint64_t n, Affine<F>* __restrict__ out, int* flag) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    constexpr int B = FieldIO<F>::BYTES;
    const uint8_t* p = in + 2 * B * i;
    out[i] = Affine<F>{FieldIO<F>::load(p, flag), FieldIO<F>::load(p + B, flag)};   // all-zero stays (0,0) = infinity
}
template <class F>
__global__ void __launch_bounds__(128) k_points_from_mont(const Affine<F>* __restrict__ in, uint64_t n, uint8_t* __restrict__ out) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    constexpr int B = FieldIO<F>::BYTES;
    Affine<F> p = in[i];
    FieldIO<F>::store(out + 2 * B * i, p.x);
    FieldIO<F>::store(out + 2 * B * i + B, p.y);
}

#ifdef OG_MSM_G1
int32_t g1_bytes_to_mont(og_ctx* ctx, const uint8_t* d_in, uint64_t n, G1Affine* d_out) {
    if (n) OG_LAUNCH(ctx, k_points_to_mont<Fq>, (unsigned)((n + 127) / 128), 128, 0, d_in, n, d_out, ctx->d_flag);
    return OG_OK;
}
#endif  // OG_MSM_G1

#ifdef OG_MSM_G2
int32_t g2_bytes_to_mont(og_ctx* ctx, const uint8_t* d_in, uint64_t n, G2Affine* d_out) {
    if (n) OG_LAUNCH(ctx, k_points_to_mont<Fq2>, (unsigned)((n + 127) / 128), 128, 0, d_in, n, d_out, ctx->d_flag);
    return OG_OK;
}
#endif  // OG_MSM_G2

#ifdef OG_MSM_G1
int32_t g1_mont_to_bytes(og_ctx* ctx, const G1Affine* d_in, uint64_t n, uint8_t* d_out) {
    if (n) OG_LAUNCH(ctx, k_points_from_mont<Fq>, (unsigned)((n + 127) / 128), 128, 0, d_in, n, d_out);
    return OG_OK;
}
#endif  // OG_MSM_G1

#ifdef OG_MSM_G2
int32_t g2_mont_to_bytes(og_ctx* ctx, const G2Affine* d_in, uint64_t n, uint8_t* d_out) {
    if (n) OG_LAUNCH(ctx, k_points_from_mont<Fq2>, (unsigned)((n + 127) / 128), 128, 0, d_in, n, d_out);
    return OG_OK;
}
#endif  // OG_MSM_G2


#ifdef OG_MSM_G1
// ---- 1/3: digits -> histogram / scatter ---------------------------------------------------------------
// Signed c-bit digits of one scalar: v = bits + carry; v > 2^(c-1) -> digit v - 2^c, carry 1.  n_windows*c >= 255
// guarantees that the top window absorbs the last carry for every scalar < r < 2^254.
struct DigitIter {
    uint32_t s[9];
    __device__ __forceinline__ bool load(const DigitPlan& P, uint32_t prob, uint64_t i, int* flag) {
        const uint32_t* sp = P.scalars + ((uint64_t)prob * P.scalar_stride + i) * 8;
        if (P.montgomery) {
            Fr v;
#pragma unroll
            for (int j = 0; j < 8; j++) v.l[j] = sp[j];
            v.to_canonical(s);
        } else {
#pragma unroll
            for (int j = 0; j < 8; j++) s[j] = sp[j];
            if (!Fr::canonical_lt_mod(s)) { atomicOr(flag, 1); return false; }
        }
        s[8] = 0;
        return (s[0] | s[1] | s[2] | s[3] | s[4] | s[5] | s[6] | s[7]) != 0;
    }
    __device__ __forceinline__ void clear() {
#pragma unroll
        for (int j = 0; j < 9; j++) s[j] = 0;
    }
    // load() in two halves, so that a loop can issue the next scalar's loads before it works on the current one
    // (32-byte aligned scalars: the prover's Fr vectors)
    static __device__ __forceinline__ void fetch(const DigitPlan& P, uint32_t prob, uint64_t i, uint32_t raw[8]) {
        const uint4* sp = reinterpret_cast<const uint4*>(P.scalars + ((uint64_t)prob * P.scalar_stride + i) * 8);
        const uint4 a = sp[0], b = sp[1];
        raw[0] = a.x; raw[1] = a.y; raw[2] = a.z; raw[3] = a.w; raw[4] = b.x; raw[5] = b.y; raw[6] = b.z; raw[7] = b.w;
    }
    __device__ __forceinline__ bool from_raw(const DigitPlan& P, const uint32_t raw[8], int* flag) {
        if (P.montgomery) {
            Fr v;
#pragma unroll
            for (int j = 0; j < 8; j++) v.l[j] = raw[j];
            v.to_canonical(s);
        } else {
#pragma unroll
            for (int j = 0; j < 8; j++) s[j] = raw[j];
            if (!Fr::canonical_lt_mod(s)) { atomicOr(flag, 1); return false; }
        }
        s[8] = 0;
        return (s[0] | s[1] | s[2] | s[3] | s[4] | s[5] | s[6] | s[7]) != 0;
    }
    // calls f(window, magnitude, negative) for every window, zero digits included
    template <class Fn>
    __device__ __forceinline__ void windows(const DigitPlan& P, Fn f) const {
        const uint32_t c = P.c, half = 1u << (c - 1), mask = (1u << c) - 1;
        uint32_t carry = 0;
        for (uint32_t w = 0; w < P.n_windows; w++) {
            uint32_t bit = w * c, word = bit >> 5, sh = bit & 31;
            uint64_t two = ((uint64_t)s[word + 1] << 32) | s[word];
            uint32_t v = ((uint32_t)(two >> sh) & mask) + carry;
            uint32_t neg = v > half;
            uint32_t mag = neg ? (1u << c) - v : v;
            carry = neg;
            f(w, mag, neg);
        }
    }
    // calls f(window, magnitude - 1, negative) for every non-zero signed digit
    template <class Fn>
    __device__ __forceinline__ void for_each(const DigitPlan& P, Fn f) const {
        windows(P, [&](uint32_t w, uint32_t mag, uint32_t neg) { if (mag) f(w, mag - 1, neg); });
    }
};

// one thread per scalar, global atomics (one-shot MSMs: up to 2^15 buckets x 16 windows of keys).  The scatter is pure
// atomic round-trip latency (warps wait on the long scoreboard); cutting eight windows first and issuing their eight atomics
// back to back does not help: the L2 atomic units, not the per-thread dependency, are what the kernel waits for.
template <bool SCATTER>
__global__ void __launch_bounds__(256) k_digits(DigitPlan P, uint32_t* __restrict__ counts, const uint32_t* __restrict__ offsets,
                                                uint32_t* __restrict__ cursor, uint32_t* __restrict__ sorted, int* flag) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t prob = blockIdx.y;
    if (i >= P.n) return;
    DigitIter it;
    if (!it.load(P, prob, i, flag)) return;
    it.for_each(P, [&](uint32_t w, uint32_t b, uint32_t neg) {
        uint32_t key = (prob * P.key_stride_problem + w * P.key_stride_window) * P.nb + b;
        if (!SCATTER) {
            atomicAdd(&counts[key], 1u);
        } else {
            uint32_t pos = atomicAdd(&cursor[key], 1u);          // cursor starts at the bucket's offset (k_scan_apply)
            sorted[pos] = (((uint32_t)i + w * P.tidx_window_stride) << 1) | neg;
        }
    });
}

// ---- 2: exclusive scan: tile sums -> scan of the tile sums (one CTA) -> tile rescan with offsets ----------
constexpr uint32_t SCAN_THREADS = 256, SCAN_PER_THREAD = 8, SCAN_TILE = SCAN_THREADS * SCAN_PER_THREAD;

__device__ __forceinline__ uint32_t block_exclusive_scan(uint32_t v, uint32_t* total) {   // 256 threads
    __shared__ uint32_t warp_sums[SCAN_THREADS / 32];
    __shared__ uint32_t block_total;
    uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    uint32_t inc = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { uint32_t t = __shfl_up_sync(0xffffffffu, inc, d); if (lane >= (uint32_t)d) inc += t; }
    if (lane == 31) warp_sums[wid] = inc;
    __syncthreads();
    if (wid == 0) {
        uint32_t w = lane < SCAN_THREADS / 32 ? warp_sums[lane] : 0, winc = w;
#pragma unroll
        for (int d = 1; d < 8; d <<= 1) { uint32_t t = __shfl_up_sync(0xffffffffu, winc, d); if (lane >= (uint32_t)d) winc += t; }
        if (lane < SCAN_THREADS / 32) warp_sums[lane] = winc - w;
        if (lane == SCAN_THREADS / 32 - 1) block_total = winc;
    }
    __syncthreads();
    uint32_t r = inc - v + warp_sums[wid];
    *total = block_total;
    __syncthreads();
    return r;
}

__global__ void __launch_bounds__(SCAN_THREADS) k_scan_tiles(const uint32_t* __restrict__ counts, uint32_t n, uint32_t* __restrict__ tile_sums) {
    uint32_t base = blockIdx.x * SCAN_TILE + threadIdx.x * SCAN_PER_THREAD, s = 0;
#pragma unroll
    for (uint32_t k = 0; k < SCAN_PER_THREAD; k++) if (base + k < n) s += counts[base + k];
    uint32_t total;
    block_exclusive_scan(s, &total);
    if (threadIdx.x == 0) tile_sums[blockIdx.x] = total;
}
// in-place exclusive scan of up to SCAN_TILE * 64 tile sums by one CTA
__global__ void __launch_bounds__(SCAN_THREADS) k_scan_tile_sums(uint32_t* __restrict__ tile_sums, uint32_t n_tiles, uint32_t* __restrict__ grand_total) {
    uint32_t run = 0;
    for (uint32_t base = 0; base < n_tiles; base += SCAN_THREADS) {
        uint32_t i = base + threadIdx.x;
        uint32_t v = i < n_tiles ? tile_sums[i] : 0, total;
        uint32_t ex = block_exclusive_scan(v, &total);
        if (i < n_tiles) tile_sums[i] = run + ex;
        run += total;
    }
    if (threadIdx.x == 0) *grand_total = run;
}
__global__ void __launch_bounds__(SCAN_THREADS) k_scan_apply(const uint32_t* __restrict__ counts, uint32_t n, const uint32_t* __restrict__ tile_sums,
                                                            uint32_t* __restrict__ offsets, uint32_t* __restrict__ cursor) {
    uint32_t base = blockIdx.x * SCAN_TILE + threadIdx.x * SCAN_PER_THREAD;
    uint32_t c[SCAN_PER_THREAD], s = 0;
#pragma unroll
    for (uint32_t k = 0; k < SCAN_PER_THREAD; k++) { c[k] = base + k < n ? counts[base + k] : 0; s += c[k]; }
    uint32_t total;
    uint32_t run = tile_sums[blockIdx.x] + block_exclusive_scan(s, &total);
#pragma unroll
    for (uint32_t k = 0; k < SCAN_PER_THREAD; k++) {      // the scatter's cursors start at the offsets: one random access per entry fewer
        if (base + k < n) { offsets[base + k] = run; if (cursor) cursor[base + k] = run; }
        run += c[k];
    }
}

// offsets[n] receives the grand total; cursor (optional) a copy of the offsets
static int32_t exclusive_scan(og_ctx* ctx, const uint32_t* d_counts, uint32_t n, uint32_t* d_offsets, uint32_t* d_cursor) {
    uint32_t n_tiles = (n + SCAN_TILE - 1) / SCAN_TILE;
    OG_SLOT(ctx, tile_sums, uint32_t, ctx->lane ? S_L1_MSM_MISC : S_MSM_MISC, 4 * (size_t)n_tiles);
    OG_LAUNCH(ctx, k_scan_tiles, n_tiles, SCAN_THREADS, 0, d_counts, n, tile_sums);
    OG_LAUNCH(ctx, k_scan_tile_sums, 1, SCAN_THREADS, 0, tile_sums, n_tiles, d_offsets + n);
    OG_LAUNCH(ctx, k_scan_apply, n_tiles, SCAN_THREADS, 0, d_counts, n, tile_sums, d_offsets, d_cursor);
    return OG_OK;
}

// ---- the batched prover's sort (one group per proof): a two-pass partitioned counting sort --------------------------------
// A scatter with one global cursor atomic per entry into 2^15 buckets per proof waits on L2 atomic round trips and writes
// 4-byte entries to random places.  Instead each proof's entries are first split into P coarse partitions (the top bits of
// the bucket id), then every partition is sorted by the remaining bits on its own:
//   k_sort_part_count    per (tile of SORT_TILE scalars, proof): digits per partition, counted in shared memory
//   exclusive_scan       of those counts in (proof, partition, tile) order: each (tile, partition) gets a run, and the runs of
//                        one (proof, partition) are adjacent -- they span that partition's window of the final list
//   k_sort_part_scatter  the digits again: entry + fine bucket id (bucket mod nb/P, one byte) into the tile's runs of a
//                        staging array, ranked by shared-memory cursors (no global atomics; runs of ~2 KB for C')
//   k_sort_local         per (proof, partition): histogram of the fine ids -> counts and offsets of the partition's buckets,
//                        then the entries into the partition's window of the list (~35 KB for C'), whose stores L2 combines
// Any digit distribution works: every loop is bounded by the tile or the partition, not by a bin's load, and lanes of a
// warp that hit the same shared counter add once (a 0/1 witness puts nearly every digit in one bucket).
// P = 128 and tiles of 4096 scalars were the fastest of the sweep in DESIGN.md section 8.
constexpr uint32_t SORT_PARTS = 128, SORT_TILE = 4096, SORT_THREADS = 256;
constexpr uint32_t SORT_MAX_NB = 32768, SORT_MAX_FINE = SORT_MAX_NB / SORT_PARTS;     // c <= 16
constexpr uint32_t NO_BIN = 0xFFFFFFFFu;
static_assert(SORT_THREADS == SCAN_THREADS, "k_sort_local scans with block_exclusive_scan");
static_assert(SORT_PARTS <= SORT_THREADS && SORT_MAX_FINE <= SORT_THREADS && SORT_TILE % SORT_THREADS == 0, "sort shape");
static_assert(SORT_MAX_FINE <= 256, "fine bucket ids are staged as one byte");

static uint32_t sort_parts(uint32_t nb) { return nb < SORT_PARTS ? nb : SORT_PARTS; }
static uint32_t sort_shift(uint32_t nb) { uint32_t s = 0; while ((sort_parts(nb) << s) < nb) s++; return s; }
static uint64_t sort_tiles(uint64_t n) { return (n + SORT_TILE - 1) / SORT_TILE; }

// Called by all 32 lanes of a warp; bin NO_BIN adds nothing.  Returns the lane's slot: the bin's old value plus the lane's
// rank in the warp.  When every lane with a bin has the same one (skewed digits: a 0/1 witness puts nearly every digit in
// one bucket), the warp adds with one atomic instead of 32 on one address; otherwise each lane adds its own (cheaper than
// grouping the lanes by bin with __match_any_sync, which made the uniform case slower).
__device__ __forceinline__ uint32_t warp_bin_add(uint32_t* bins, uint32_t bin) {
    const uint32_t lane = threadIdx.x & 31, valid = __ballot_sync(0xffffffffu, bin != NO_BIN);
    if (!valid) return 0;
    const uint32_t leader = __ffs(valid) - 1, first = __shfl_sync(0xffffffffu, bin, leader);
    if (__all_sync(0xffffffffu, bin == NO_BIN || bin == first)) {
        uint32_t base = 0;
        if (lane == leader) base = atomicAdd(&bins[first], (uint32_t)__popc(valid));
        return __shfl_sync(0xffffffffu, base, leader) + __popc(valid & ((1u << lane) - 1));
    }
    return bin != NO_BIN ? atomicAdd(&bins[bin], 1u) : 0;
}

// tile_counts[(proof * parts + partition) * n_tiles + tile]
__global__ void __launch_bounds__(SORT_THREADS) k_sort_part_count(DigitPlan P, uint32_t shift, uint32_t n_tiles,
                                                                  uint32_t* __restrict__ tile_counts, int* flag) {
    __shared__ uint32_t hist[SORT_PARTS];
    const uint32_t prob = blockIdx.y, tile = blockIdx.x, parts = P.nb >> shift;
    for (uint32_t p = threadIdx.x; p < parts; p += SORT_THREADS) hist[p] = 0;
    __syncthreads();
    const uint64_t lo = (uint64_t)tile * SORT_TILE, hi = lo + SORT_TILE < P.n ? lo + SORT_TILE : P.n;
    uint32_t raw[8];
    if (lo + threadIdx.x < hi) DigitIter::fetch(P, prob, lo + threadIdx.x, raw);
    for (uint64_t i0 = lo; i0 < hi; i0 += SORT_THREADS) {          // the same trip count for every lane: warp_bin_add needs all 32
        const uint64_t i = i0 + threadIdx.x;
        DigitIter it;
        if (!(i < hi && it.from_raw(P, raw, flag))) it.clear();
        if (i + SORT_THREADS < hi) DigitIter::fetch(P, prob, i + SORT_THREADS, raw);     // in flight while this scalar is cut
        it.windows(P, [&](uint32_t, uint32_t mag, uint32_t) { warp_bin_add(hist, mag ? (mag - 1) >> shift : NO_BIN); });
    }
    __syncthreads();
    for (uint32_t p = threadIdx.x; p < parts; p += SORT_THREADS) tile_counts[((size_t)prob * parts + p) * n_tiles + tile] = hist[p];
}

// tile_offs: exclusive scan of tile_counts = where the (proof, partition, tile) run starts in the staging (and in the list).
// Written straight from the digit loop, every lane's store went to another partition (32 sectors per warp store): the kernel
// was slower than the atomic scatter it replaces.  So each round of SORT_THREADS scalars (up to SORT_ROUND_WINDOWS windows)
// is first ordered by partition in shared memory and then copied out: consecutive lanes store consecutive slots of a run.
constexpr uint32_t SORT_ROUND_WINDOWS = 24, SORT_ROUND = SORT_THREADS * SORT_ROUND_WINDOWS;   // 36 KB per round: 5 CTAs per SM
__global__ void __launch_bounds__(SORT_THREADS) k_sort_part_scatter(DigitPlan P, uint32_t shift, uint32_t n_tiles,
                                                                    const uint32_t* __restrict__ tile_offs, uint32_t* __restrict__ stage_e,
                                                                    uint8_t* __restrict__ stage_f, int* flag) {
    __shared__ uint32_t sm_e[SORT_ROUND];
    __shared__ uint16_t sm_b[SORT_ROUND];                           // bucket (< nb <= 2^15)
    __shared__ uint32_t cnt[SORT_PARTS], lbase[SORT_PARTS], cur[SORT_PARTS];
    const uint32_t tid = threadIdx.x, prob = blockIdx.y, tile = blockIdx.x, parts = P.nb >> shift, fmask = (1u << shift) - 1;
    for (uint32_t p = tid; p < parts; p += SORT_THREADS) { cur[p] = tile_offs[((size_t)prob * parts + p) * n_tiles + tile]; cnt[p] = 0; }
    __syncthreads();
    const uint64_t lo = (uint64_t)tile * SORT_TILE, hi = lo + SORT_TILE < P.n ? lo + SORT_TILE : P.n;
    uint32_t raw[8];
    if (lo + tid < hi) DigitIter::fetch(P, prob, lo + tid, raw);
    for (uint64_t i0 = lo; i0 < hi; i0 += SORT_THREADS) {
        const uint64_t i = i0 + tid;
        DigitIter it;
        if (!(i < hi && it.from_raw(P, raw, flag))) it.clear();
        if (i + SORT_THREADS < hi) DigitIter::fetch(P, prob, i + SORT_THREADS, raw);     // in flight during the round
        for (uint32_t w0 = 0; w0 < P.n_windows; w0 += SORT_ROUND_WINDOWS) {
            auto bin_of = [&](uint32_t w, uint32_t mag) { return mag && w >= w0 && w < w0 + SORT_ROUND_WINDOWS ? (mag - 1) >> shift : NO_BIN; };
            it.windows(P, [&](uint32_t w, uint32_t mag, uint32_t) { warp_bin_add(cnt, bin_of(w, mag)); });
            __syncthreads();
            uint32_t n_round, b = block_exclusive_scan(tid < parts ? cnt[tid] : 0, &n_round);
            if (tid < parts) { lbase[tid] = b; cnt[tid] = b; }      // cnt: the round's cursors from here on
            __syncthreads();
            it.windows(P, [&](uint32_t w, uint32_t mag, uint32_t neg) {
                const uint32_t bin = bin_of(w, mag), pos = warp_bin_add(cnt, bin);
                if (bin != NO_BIN) { sm_e[pos] = (((uint32_t)i + w * P.tidx_window_stride) << 1) | neg; sm_b[pos] = (uint16_t)(mag - 1); }
            });
            __syncthreads();
            for (uint32_t k = tid; k < n_round; k += SORT_THREADS) {
                const uint32_t bk = sm_b[k], p = bk >> shift, dst = cur[p] + k - lbase[p];
                stage_e[dst] = sm_e[k];
                stage_f[dst] = (uint8_t)(bk & fmask);
            }
            __syncthreads();
            if (tid < parts) { cur[tid] += cnt[tid] - lbase[tid]; cnt[tid] = 0; }
            __syncthreads();
        }
    }
}

// one CTA per (proof, partition) g; its buckets are keys g * 2^shift + f.  A partition of up to SORT_LOCAL_CAP entries is
// assembled in shared memory and written out in order; a larger one (skewed digits) is scattered straight into the list.
// Each thread loads SORT_LOCAL_ITEMS entries before it ranks any of them: with one load per rank the kernel waited on
// memory latency.
constexpr uint32_t SORT_LOCAL_CAP = 10240;                          // 40 KB (5 CTAs per SM); C' partitions average ~8.7k entries
constexpr uint32_t SORT_LOCAL_ITEMS = 8, SORT_LOCAL_STEP = SORT_THREADS * SORT_LOCAL_ITEMS;
__global__ void __launch_bounds__(SORT_THREADS) k_sort_local(const uint32_t* __restrict__ tile_offs, uint32_t n_tiles, uint32_t n_parts,
                                                             uint32_t shift, const uint32_t* __restrict__ total,
                                                             const uint32_t* __restrict__ stage_e, const uint8_t* __restrict__ stage_f,
                                                             uint32_t* __restrict__ counts, uint32_t* __restrict__ offsets,
                                                             uint32_t* __restrict__ sorted) {
    __shared__ uint32_t bins[SORT_THREADS];                         // >= SORT_MAX_FINE fine buckets
    __shared__ uint32_t sm_out[SORT_LOCAL_CAP];
    const uint32_t g = blockIdx.x, F = 1u << shift, tid = threadIdx.x;
    const uint32_t start = tile_offs[(size_t)g * n_tiles], end = g + 1 < n_parts ? tile_offs[(size_t)(g + 1) * n_tiles] : *total;
    if (g + 1 == n_parts && tid == 0) offsets[(size_t)n_parts * F] = end;          // offsets[n_keys] = the total
    bins[tid] = 0;
    __syncthreads();
    for (uint32_t j0 = start; j0 < end; j0 += SORT_LOCAL_STEP) {
        uint32_t f[SORT_LOCAL_ITEMS];
#pragma unroll
        for (uint32_t k = 0; k < SORT_LOCAL_ITEMS; k++) { const uint32_t j = j0 + k * SORT_THREADS + tid; f[k] = j < end ? stage_f[j] : NO_BIN; }
#pragma unroll
        for (uint32_t k = 0; k < SORT_LOCAL_ITEMS; k++) warp_bin_add(bins, f[k]);
    }
    __syncthreads();
    const uint32_t c = tid < F ? bins[tid] : 0;
    uint32_t tot;
    const uint32_t run = start + block_exclusive_scan(c, &tot);      // (ends with a barrier: every bin has been read)
    if (tid < F) {
        const size_t key = (size_t)g * F + tid;
        counts[key] = c; offsets[key] = run; bins[tid] = run;
    }
    __syncthreads();
    const bool staged = end - start <= SORT_LOCAL_CAP;             // the same for the whole CTA
    for (uint32_t j0 = start; j0 < end; j0 += SORT_LOCAL_STEP) {
        uint32_t f[SORT_LOCAL_ITEMS], e[SORT_LOCAL_ITEMS];
#pragma unroll
        for (uint32_t k = 0; k < SORT_LOCAL_ITEMS; k++) {
            const uint32_t j = j0 + k * SORT_THREADS + tid;
            f[k] = j < end ? stage_f[j] : NO_BIN;
            e[k] = j < end ? stage_e[j] : 0;
        }
#pragma unroll
        for (uint32_t k = 0; k < SORT_LOCAL_ITEMS; k++) {
            const uint32_t pos = warp_bin_add(bins, f[k]);
            if (f[k] != NO_BIN) { if (staged) sm_out[pos - start] = e[k]; else sorted[pos] = e[k]; }
        }
    }
    if (staged) {
        __syncthreads();
        for (uint32_t k = tid; k < end - start; k += SORT_THREADS) sorted[start + k] = sm_out[k];
    }
}

size_t msm_sort_stage_bytes(uint64_t n_entries) { return 5 * n_entries; }
size_t msm_sort_tile_bytes(uint32_t n_problems, uint32_t nb, uint64_t n) { return 8 * (size_t)n_problems * sort_parts(nb) * sort_tiles(n) + 4; }

int32_t msm_sort_digits(og_ctx* ctx, const DigitPlan& plan, uint32_t n_keys, uint32_t* d_counts, uint32_t* d_offsets,
                        uint32_t* d_cursor, uint32_t* d_sorted, uint32_t* d_stage, uint32_t* d_tiles) {
    if (plan.n == 0 || plan.n_problems == 0) {
        OG_CUDA(ctx, cudaMemsetAsync(d_counts, 0, sizeof(uint32_t) * (size_t)n_keys, ctx->stream));
        OG_CUDA(ctx, cudaMemsetAsync(d_offsets, 0, sizeof(uint32_t) * ((size_t)n_keys + 1), ctx->stream));
        return OG_OK;
    }
    if (plan.key_stride_window == 0) {            // batched prover: one group per proof
        if (!d_stage || !d_tiles || plan.key_stride_problem != 1 || plan.nb > SORT_MAX_NB || n_keys != plan.n_problems * plan.nb) return OG_E_INVALID;
        const uint32_t parts = sort_parts(plan.nb), shift = sort_shift(plan.nb), n_tiles = (uint32_t)sort_tiles(plan.n);
        const uint32_t n_parts = plan.n_problems * parts, n_runs = n_parts * n_tiles;
        uint32_t* tile_counts = d_tiles;
        uint32_t* tile_offs = d_tiles + n_runs;       // n_runs + 1 (the grand total)
        uint32_t* stage_e = d_stage;
        uint8_t* stage_f = reinterpret_cast<uint8_t*>(d_stage + (uint64_t)plan.n_problems * plan.n * plan.n_windows);
        dim3 tgrid(n_tiles, plan.n_problems);
        OG_LAUNCH(ctx, k_sort_part_count, tgrid, SORT_THREADS, 0, plan, shift, n_tiles, tile_counts, ctx->d_flag);
        OG_TRY(exclusive_scan(ctx, tile_counts, n_runs, tile_offs, nullptr));
        OG_LAUNCH(ctx, k_sort_part_scatter, tgrid, SORT_THREADS, 0, plan, shift, n_tiles, tile_offs, stage_e, stage_f, ctx->d_flag);
        OG_LAUNCH(ctx, k_sort_local, n_parts, SORT_THREADS, 0, tile_offs, n_tiles, n_parts, shift, tile_offs + n_runs, stage_e, stage_f,
                  d_counts, d_offsets, d_sorted);
        return OG_OK;
    }
    OG_CUDA(ctx, cudaMemsetAsync(d_counts, 0, sizeof(uint32_t) * (size_t)n_keys, ctx->stream));
    dim3 grid((unsigned)((plan.n + 255) / 256), plan.n_problems);
    OG_LAUNCHN(ctx, "k_digits_count", k_digits<false>, grid, 256, 0, plan, d_counts, nullptr, nullptr, nullptr, ctx->d_flag);
    OG_TRY(exclusive_scan(ctx, d_counts, n_keys, d_offsets, d_cursor));
    OG_LAUNCHN(ctx, "k_digits_scatter", k_digits<true>, grid, 256, 0, plan, d_counts, d_offsets, d_cursor, d_sorted, ctx->d_flag);
    return OG_OK;
}
#endif  // OG_MSM_G1


// ---- 3b: order the buckets of every group by decreasing load ------------------------------------------------
// Bucket loads are Poisson-distributed, so a warp of 32 neighbouring buckets waits for its longest list
// (ncu shows a quarter or more of the lanes idle).  A counting sort of the bucket ids by their count
// puts equal loads in the same warp and schedules the longest lists first.
constexpr uint32_t ORDER_BINS = 2048;
template <class F>   // (template only so that each translation unit gets its own copy)
__global__ void __launch_bounds__(1024) k_bucket_order(const uint32_t* __restrict__ counts, uint32_t nb, uint32_t* __restrict__ perm) {
    __shared__ uint32_t hist[ORDER_BINS];
    const uint32_t g = blockIdx.x, t = threadIdx.x;
    const uint32_t* c = counts + (size_t)g * nb;
    for (uint32_t i = t; i < ORDER_BINS; i += 1024) hist[i] = 0;
    __syncthreads();
    for (uint32_t b = t; b < nb; b += 1024) atomicAdd(&hist[ORDER_BINS - 1 - min(c[b], ORDER_BINS - 1)], 1u);
    __syncthreads();
    // exclusive scan of 2048 bins by 1024 threads (two bins each) + Hillis-Steele over the pair sums
    __shared__ uint32_t pair[1024];
    uint32_t a0 = hist[2 * t], a1 = hist[2 * t + 1];
    pair[t] = a0 + a1;
    __syncthreads();
    for (uint32_t d = 1; d < 1024; d <<= 1) {
        uint32_t v = t >= d ? pair[t - d] : 0;
        __syncthreads();
        pair[t] += v;
        __syncthreads();
    }
    uint32_t base = t ? pair[t - 1] : 0;
    hist[2 * t] = base;
    hist[2 * t + 1] = base + a0;
    __syncthreads();
    for (uint32_t b = t; b < nb; b += 1024) {
        uint32_t pos = atomicAdd(&hist[ORDER_BINS - 1 - min(c[b], ORDER_BINS - 1)], 1u);
        perm[(size_t)g * nb + pos] = g * nb + b;
    }
}

// ---- 4: bucket accumulation ----------------------------------------------------------------------------
template <class F>
__device__ __forceinline__ Affine<F> fetch_point(const Affine<F>* __restrict__ table, uint32_t e) {
    Affine<F> p = table[e >> 1];
    if (e & 1) p.y = p.y.neg();
    return p;
}

#ifdef OG_MSM_G1
// G1 variant with the 128-byte accumulator in shared memory (see the G2 one below): 8 chunks of 16 bytes per thread.
struct SmAcc1 {
    uint4* base;    // [8 chunks][128 threads]
    __device__ __forceinline__ Fq ld(int coord) const {
        Fq v;
        uint4 a = base[(coord * 2 + 0) * 128], b = base[(coord * 2 + 1) * 128];
        v.l[0] = a.x; v.l[1] = a.y; v.l[2] = a.z; v.l[3] = a.w; v.l[4] = b.x; v.l[5] = b.y; v.l[6] = b.z; v.l[7] = b.w;
        return v;
    }
    __device__ __forceinline__ void st(int coord, const Fq& v) const {
        base[(coord * 2 + 0) * 128] = make_uint4(v.l[0], v.l[1], v.l[2], v.l[3]);
        base[(coord * 2 + 1) * 128] = make_uint4(v.l[4], v.l[5], v.l[6], v.l[7]);
    }
};

// 8 CTAs of 128 threads per SM (64 registers); only the next 4-byte ENTRY is read ahead, the 64-byte gather is
// covered by the other warps (compared against 6/7 CTAs and against a prefetched point)
// the two squarings of a mixed addition through ONE out-of-line copy of the wide squarer (8 registers in, 8 out): with the squarer
// inlined twice next to eight inlined products the kernel outgrows the instruction cache (ncu: warps waiting for instructions)
#ifndef OG_SQR_CALL
#define OG_SQR_CALL 1
#endif
#if OG_SQR_CALL
static __device__ __noinline__ Fq fq_sqr_call(Fq a) { return a.sqr(); }
#define OG_ACC_SQR(x) fq_sqr_call(x)
#else
#define OG_ACC_SQR(x) (x).sqr()
#endif
#if defined(OG_MUL_CALL) && OG_MUL_CALL      // A/B: the eight products out of line as well
static __device__ __noinline__ Fq fq_mul_call(Fq a, Fq b) { return a * b; }
#define OG_ACC_MUL(x, y) fq_mul_call((x), (y))
#else
#define OG_ACC_MUL(x, y) ((x) * (y))
#endif
#ifndef OG_ACC1_MINB
#define OG_ACC1_MINB 8
#endif
__global__ void __launch_bounds__(128, OG_ACC1_MINB) k_bucket_acc_sm1(const Affine<Fq>* __restrict__ table, const uint32_t* __restrict__ sorted,
                                                        const uint32_t* __restrict__ offsets, const uint32_t* __restrict__ counts,
                                                        uint32_t n_keys, uint32_t cap, XYZZ<Fq>* __restrict__ buckets,
                                                        uint32_t* __restrict__ heavy, const uint32_t* __restrict__ perm) {
    __shared__ uint4 sm_acc[8 * 128];
    uint32_t slot_ = blockIdx.x * blockDim.x + threadIdx.x;
    if (slot_ >= n_keys) return;
    uint32_t key = perm[slot_];
    uint32_t cnt = counts[key], off = offsets[key];
    if (cnt > cap) {                               // left to k_bucket_heavy
        uint32_t slot = atomicAdd(heavy, 1u);
        heavy[1 + slot] = key;
        buckets[key] = XYZZ<Fq>::inf();
        return;
    }
    SmAcc1 A{sm_acc + threadIdx.x};
    bool inf = true;
    uint32_t e = cnt ? sorted[off] : 0;
    for (uint32_t k = 0; k < cnt; k++) {
        uint32_t en = k + 1 < cnt ? sorted[off + k + 1] : 0;
        Affine<Fq> q = fetch_point(table, e);
        e = en;
        if (q.is_inf()) continue;
        if (inf) { A.st(0, q.x); A.st(1, q.y); A.st(2, Fq::one()); A.st(3, Fq::one()); inf = false; continue; }
        Fq p = OG_ACC_MUL(q.x, A.ld(2)) - A.ld(0);
        Fq r = OG_ACC_MUL(q.y, A.ld(3)) - A.ld(1);
        if (p.is_zero()) {
            if (r.is_zero()) { XYZZ<Fq> d = XYZZ<Fq>::dbl_affine(q); A.st(0, d.x); A.st(1, d.y); A.st(2, d.zz); A.st(3, d.zzz); }
            else inf = true;
            continue;
        }
        // ordered so that few temporaries are live at a time: zz and zzz are updated as soon as pp / ppp exist
        Fq pp = OG_ACC_SQR(p);
        A.st(2, OG_ACC_MUL(A.ld(2), pp));
        Fq ppp = OG_ACC_MUL(p, pp);
        A.st(3, OG_ACC_MUL(A.ld(3), ppp));
        Fq q1 = OG_ACC_MUL(A.ld(0), pp);
        Fq x3 = OG_ACC_SQR(r) - ppp - q1.dbl();
        A.st(0, x3);
        A.st(1, OG_ACC_MUL(r, q1 - x3) - OG_ACC_MUL(A.ld(1), ppp));
    }
    buckets[key] = inf ? XYZZ<Fq>::inf() : XYZZ<Fq>{A.ld(0), A.ld(1), A.ld(2), A.ld(3)};
}

// Test/debug probe (og_field_probe_raw, unit 0): raw Montgomery limbs in and out, no conversion and no range check, through the
// product and the squarer (fq_sqr_call) of k_bucket_acc_sm1, with its launch bounds.  In this whole-program build ptxas compiles a
// copy of every __noinline__ callee into each kernel that calls it, so the probe runs its own copy of fq_sqr_call: the same PTX, but
// not necessarily the bucket kernel's register allocation.  op 0: a * b, 1: sqr(a), 2: a - b, 3: a.dbl()
__global__ void __launch_bounds__(128, OG_ACC1_MINB) k_field_probe_g1(int32_t op, const Fq* __restrict__ a, const Fq* __restrict__ b, uint64_t n,
                                                        Fq* __restrict__ out) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const Fq x = a[i], y = b[i];
    out[i] = op == 0 ? OG_ACC_MUL(x, y) : op == 1 ? OG_ACC_SQR(x) : op == 2 ? x - y : x.dbl();
}
int32_t field_probe_raw_g1(og_ctx* ctx, int32_t op, const uint8_t* d_a, const uint8_t* d_b, uint64_t n, uint8_t* d_out) {
    if (n) OG_LAUNCH(ctx, k_field_probe_g1, (unsigned)((n + 127) / 128), 128, 0, op, reinterpret_cast<const Fq*>(d_a),
                     reinterpret_cast<const Fq*>(d_b), n, reinterpret_cast<Fq*>(d_out));
    return OG_OK;
}
#endif

#ifdef OG_MSM_G2
// G2 variant with the 256-byte accumulator in shared memory (16-byte chunks interleaved over the CTA's threads, so
// every access is conflict-free).  The mixed addition is g2_madd_lazy (ec.cuh): lazily reduced Fq2 through one out-of-line copy
// of the lazy product and squaring; the accumulator stays in [0, 2p) and is made canonical when the bucket is stored.  4 resident
// CTAs (128 registers) beat 6 (80 registers, whose multiplier spilled around every call): 116.7 vs 139.6 ms per prover step.
struct SmAcc {
    uint4* base;    // [16 chunks][128 threads]
    __device__ __forceinline__ Fq2 ld(int coord) const {
        Fq2 v;
        uint4 a = base[(coord * 4 + 0) * 128], b = base[(coord * 4 + 1) * 128], c = base[(coord * 4 + 2) * 128], d = base[(coord * 4 + 3) * 128];
        v.c0.l[0] = a.x; v.c0.l[1] = a.y; v.c0.l[2] = a.z; v.c0.l[3] = a.w; v.c0.l[4] = b.x; v.c0.l[5] = b.y; v.c0.l[6] = b.z; v.c0.l[7] = b.w;
        v.c1.l[0] = c.x; v.c1.l[1] = c.y; v.c1.l[2] = c.z; v.c1.l[3] = c.w; v.c1.l[4] = d.x; v.c1.l[5] = d.y; v.c1.l[6] = d.z; v.c1.l[7] = d.w;
        return v;
    }
    __device__ __forceinline__ void st(int coord, const Fq2& v) const {
        base[(coord * 4 + 0) * 128] = make_uint4(v.c0.l[0], v.c0.l[1], v.c0.l[2], v.c0.l[3]);
        base[(coord * 4 + 1) * 128] = make_uint4(v.c0.l[4], v.c0.l[5], v.c0.l[6], v.c0.l[7]);
        base[(coord * 4 + 2) * 128] = make_uint4(v.c1.l[0], v.c1.l[1], v.c1.l[2], v.c1.l[3]);
        base[(coord * 4 + 3) * 128] = make_uint4(v.c1.l[4], v.c1.l[5], v.c1.l[6], v.c1.l[7]);
    }
};

#ifndef OG_ACC2_MINB
#define OG_ACC2_MINB 4
#endif
__global__ void __launch_bounds__(128, OG_ACC2_MINB) k_bucket_acc_sm(const Affine<Fq2>* __restrict__ table, const uint32_t* __restrict__ sorted,
                                                       const uint32_t* __restrict__ offsets, const uint32_t* __restrict__ counts,
                                                       uint32_t n_keys, uint32_t cap, XYZZ<Fq2>* __restrict__ buckets,
                                                       uint32_t* __restrict__ heavy, const uint32_t* __restrict__ perm) {
    __shared__ uint4 sm_acc[16 * 128];
    uint32_t slot_ = blockIdx.x * blockDim.x + threadIdx.x;
    if (slot_ >= n_keys) return;
    uint32_t key = perm[slot_];
    uint32_t cnt = counts[key], off = offsets[key];
    if (cnt > cap) {                               // left to k_bucket_heavy
        uint32_t slot = atomicAdd(heavy, 1u);
        heavy[1 + slot] = key;
        buckets[key] = XYZZ<Fq2>::inf();
        return;
    }
    SmAcc A{sm_acc + threadIdx.x};
    bool inf = true;
    uint32_t e = cnt ? sorted[off] : 0;
    for (uint32_t k = 0; k < cnt; k++) {
        uint32_t en = k + 1 < cnt ? sorted[off + k + 1] : 0;
        Affine<Fq2> q = fetch_point(table, e);
        e = en;
        if (q.is_inf()) continue;
        if (inf) { A.st(0, q.x); A.st(1, q.y); A.st(2, Fq2::one()); A.st(3, Fq2::one()); inf = false; continue; }
        if (!g2_madd_lazy(A, q)) inf = true;          // the accumulator stays lazy ([0, 2p)) until the bucket is stored
    }
    buckets[key] = inf ? XYZZ<Fq2>::inf() : XYZZ<Fq2>{A.ld(0).canonical(), A.ld(1).canonical(), A.ld(2).canonical(), A.ld(3).canonical()};
}

// Test/debug probe (og_field_probe_raw, unit 1): raw Montgomery limbs in and out, no conversion and no range check, through the
// lazy and canonical Fq2 products of this unit (fq2_mul_lazy_call, fq2_sqr_lazy_call, fq2_mul_call, fq2_sqr_call), with
// k_bucket_acc_sm's launch bounds.  Like every kernel of this build, the probe gets its own ptxas copy of those callees: the same PTX
// as the bucket kernel's, not necessarily the same register allocation.  op 0: fq2_mul_lazy, 1: fq2_sqr_lazy, 2: add_lazy, 3: sub_lazy,
// 4: canonical(a), 5: a * b, 6: a.sqr(), 7: is_zero_lazy(a) (1 or 0 in limb 0 of c0, every other limb 0)
__global__ void __launch_bounds__(128, OG_ACC2_MINB) k_field_probe_g2(int32_t op, const Fq2* __restrict__ a, const Fq2* __restrict__ b, uint64_t n,
                                                        Fq2* __restrict__ out) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const Fq2 x = a[i], y = b[i];
    Fq2 z;
    switch (op) {
        case 0: z = fq2_mul_lazy(x, y); break;
        case 1: z = fq2_sqr_lazy(x); break;
        case 2: z = Fq2::add_lazy(x, y); break;
        case 3: z = Fq2::sub_lazy(x, y); break;
        case 4: z = x.canonical(); break;
        case 5: z = x * y; break;
        case 6: z = x.sqr(); break;
        default: z = Fq2::zero(); z.c0.l[0] = x.is_zero_lazy() ? 1u : 0u; break;
    }
    out[i] = z;
}
int32_t field_probe_raw_g2(og_ctx* ctx, int32_t op, const uint8_t* d_a, const uint8_t* d_b, uint64_t n, uint8_t* d_out) {
    if (n) OG_LAUNCH(ctx, k_field_probe_g2, (unsigned)((n + 127) / 128), 128, 0, op, reinterpret_cast<const Fq2*>(d_a),
                     reinterpret_cast<const Fq2*>(d_b), n, reinterpret_cast<Fq2*>(d_out));
    return OG_OK;
}
#endif

// Heavy buckets (lists above the cap: witness-like scalars put 30 % of all points into bucket "1" of window 0) are cut
// into segments of `seg` entries; every segment gets a CTA, a second kernel adds the partial sums of each bucket.
// (One CTA per whole list left 3*10^5 entries of a witness-like 2^20 MSM on 256 threads.)
// heavy[0] = number of heavy buckets, heavy[1 ..] = their keys, heavy[1 + n_keys ..] = first segment of each (+ total).
template <class F>   // (template only so that each translation unit gets its own copy)
__global__ void __launch_bounds__(256) k_heavy_plan(uint32_t* __restrict__ heavy, const uint32_t* __restrict__ counts, uint32_t n_keys, uint32_t seg) {
    __shared__ uint32_t part[256];
    __shared__ uint32_t carry;
    const uint32_t n_heavy = heavy[0];
    uint32_t* seg_base = heavy + 1 + n_keys;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (uint32_t base = 0; base < n_heavy; base += 256) {
        uint32_t h = base + threadIdx.x;
        uint32_t v = h < n_heavy ? (counts[heavy[1 + h]] + seg - 1) / seg : 0;
        part[threadIdx.x] = v;
        __syncthreads();
        for (uint32_t d = 1; d < 256; d <<= 1) {
            uint32_t t = threadIdx.x >= d ? part[threadIdx.x - d] : 0;
            __syncthreads();
            part[threadIdx.x] += t;
            __syncthreads();
        }
        if (h < n_heavy) seg_base[h] = carry + part[threadIdx.x] - v;
        __syncthreads();
        if (threadIdx.x == 255) carry += part[255];
        __syncthreads();
    }
    if (threadIdx.x == 0) seg_base[n_heavy] = carry;
}

template <class F, int THREADS>
__global__ void __launch_bounds__(THREADS) k_bucket_heavy(const Affine<F>* __restrict__ table, const uint32_t* __restrict__ sorted,
                                                          const uint32_t* __restrict__ offsets, const uint32_t* __restrict__ counts,
                                                          uint32_t n_keys, uint32_t seg, XYZZ<F>* __restrict__ partials,
                                                          const uint32_t* __restrict__ heavy) {
    extern __shared__ __align__(32) unsigned char smem_raw[];
    XYZZ<F>* sh = reinterpret_cast<XYZZ<F>*>(smem_raw);
    const uint32_t n_heavy = heavy[0];
    const uint32_t* seg_base = heavy + 1 + n_keys;
    const uint32_t n_seg = n_heavy ? seg_base[n_heavy] : 0;
    for (uint32_t g = blockIdx.x; g < n_seg; g += gridDim.x) {
        uint32_t lo = 0, hi = n_heavy;                          // largest h with seg_base[h] <= g
        while (hi - lo > 1) { uint32_t mid = (lo + hi) >> 1; if (seg_base[mid] <= g) lo = mid; else hi = mid; }
        const uint32_t key = heavy[1 + lo];
        const uint32_t cnt = counts[key], off = offsets[key];
        const uint32_t k0 = (g - seg_base[lo]) * seg, k1 = k0 + seg < cnt ? k0 + seg : cnt;
        XYZZ<F> acc = XYZZ<F>::inf();
        for (uint32_t k = k0 + threadIdx.x; k < k1; k += THREADS) { Affine<F> q = fetch_point(table, sorted[off + k]); xyzz_madd_ni(&acc, &q); }
        sh[threadIdx.x] = acc;
        __syncthreads();
        for (int s = THREADS / 2; s > 0; s >>= 1) {
            if ((int)threadIdx.x < s) xyzz_add_ni(&sh[threadIdx.x], &sh[threadIdx.x + s]);
            __syncthreads();
        }
        if (threadIdx.x == 0) partials[g] = sh[0];
        __syncthreads();
    }
}

// buckets[key] = sum of the bucket's segment sums (one warp per heavy bucket)
template <class F>
__global__ void __launch_bounds__(32) k_heavy_combine(const XYZZ<F>* __restrict__ partials, uint32_t n_keys, XYZZ<F>* __restrict__ buckets,
                                                      const uint32_t* __restrict__ heavy) {
    __shared__ XYZZ<F> sh[32];
    const uint32_t n_heavy = heavy[0];
    const uint32_t* seg_base = heavy + 1 + n_keys;
    for (uint32_t h = blockIdx.x; h < n_heavy; h += gridDim.x) {
        const uint32_t s0 = seg_base[h], s1 = seg_base[h + 1];
        XYZZ<F> acc = XYZZ<F>::inf();
        for (uint32_t s = s0 + threadIdx.x; s < s1; s += 32) xyzz_add_ni(&acc, &partials[s]);
        sh[threadIdx.x] = acc;
        __syncwarp();
        for (int w = 16; w > 0; w >>= 1) {
            if ((int)threadIdx.x < w) xyzz_add_ni(&sh[threadIdx.x], &sh[threadIdx.x + w]);
            __syncwarp();
        }
        if (threadIdx.x == 0) buckets[heavy[1 + h]] = sh[0];
        __syncwarp();
    }
}

#ifdef OG_EXPERIMENT_AFFINE
#include "experiments/bucket_affine.cuh"      // rejected experiment; not in the shipped library
#endif

constexpr uint32_t RED_FAN_LOG2 = 3, RED_FAN = 1u << RED_FAN_LOG2;   // 8 children per parent: more threads, shorter chains
// ---- 5: weighted reduction, RED_FAN children per parent -------------------------------------------------------
// Element e of a level carries S_e (plain sum of the buckets under e) and U_e (their 0-based weighted sum
// relative to e's first bucket).  Merging children c_0..c_k, each covering 2^w_log2 buckets:
//   S_p = sum S_c;   U_p = sum U_c + 2^w_log2 * sum_c idx(c) * S_c   (running-sum trick for the last term).
// HAS_U = false is level 0 (children are raw buckets, no weighted part yet): most of the work, and one 4-coordinate
// accumulator fewer to keep in registers.  (A variant with R and T in shared memory -- 128 instead of 226 registers,
// twice the resident warps -- was slower for G1: the R -> T chain, not occupancy, is what this kernel waits on.)
// Group operations of the reduction.  G1: ONE out-of-line copy of add and dbl with operands and result in registers (by
// value): the fully inlined kernel (three adds and a doubling, ~13k instructions) stalls waiting for instructions (ncu) at
// 8 resident warps per SM.  G2 keeps the inlined group law over the
// out-of-line Fq2 multiplier (128 registers of arguments would not travel in registers).
template <class F> struct RedOps {
    static __device__ __forceinline__ void add(XYZZ<F>& a, const XYZZ<F>& b) { a.add(b); }
    static __device__ __forceinline__ void dbl(XYZZ<F>& a) { a = a.dbl(); }
};
#ifdef OG_MSM_G1
static __device__ __noinline__ XYZZ<Fq> g1_add_rv(XYZZ<Fq> a, XYZZ<Fq> b) { a.add(b); return a; }
static __device__ __noinline__ XYZZ<Fq> g1_dbl_rv(XYZZ<Fq> a) { return a.dbl(); }
template <> struct RedOps<Fq> {
    static __device__ __forceinline__ void add(XYZZ<Fq>& a, const XYZZ<Fq>& b) { a = g1_add_rv(a, b); }
    static __device__ __forceinline__ void dbl(XYZZ<Fq>& a) { a = g1_dbl_rv(a); }
};
#endif

// G1 is faster with registers and out-of-line ops, G2 (whose register version spills) with shared memory
template <class F> constexpr bool RED_SM_DEFAULT = sizeof(F) != 32;

// (64 threads, 206 registers for G1: 4 resident CTAs per SM; asking ptxas for 6 or 8 costs spills and time)
template <class F, bool HAS_U>
__global__ void __launch_bounds__(64) k_reduce_level(const XYZZ<F>* __restrict__ S_in, const XYZZ<F>* __restrict__ U_in,
                                                     uint32_t n_in, uint32_t n_out, uint32_t n_groups, uint32_t w_log2,
                                                     uint32_t fan_log2, XYZZ<F>* __restrict__ S_out, XYZZ<F>* __restrict__ U_out) {
    uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_groups * n_out) return;
    uint32_t g = t / n_out, p = t % n_out;
    const XYZZ<F>* S = S_in + (size_t)g * n_in;
    uint32_t lo = p << fan_log2, hi = min(n_in, lo + (1u << fan_log2));
    XYZZ<F> R = XYZZ<F>::inf(), T = XYZZ<F>::inf();
    for (uint32_t i = hi - 1; i > lo; i--) {
        RedOps<F>::add(R, S[i]);
        RedOps<F>::add(T, R);
    }
    RedOps<F>::add(R, S[lo]);
    for (uint32_t k = 0; k < w_log2; k++) RedOps<F>::dbl(T);
    if (HAS_U) {
        const XYZZ<F>* U = U_in + (size_t)g * n_in;
        for (uint32_t i = lo; i < hi; i++) RedOps<F>::add(T, U[i]);
    }
    S_out[(size_t)g * n_out + p] = R;
    U_out[(size_t)g * n_out + p] = T;
}

// ---- the same level with the running sums R and T in shared memory -----------------------------------------------------
// G2: R, T and one addend are 192 registers before a single temporary, so the register version spills 2.4-3 KB per thread
// (706 LDL / 586 STL in its SASS).  Here R and T live in shared memory (16-byte chunks interleaved over the CTA's 64 threads:
// conflict-free), addend coordinates are fetched where the formula uses them, and only the temporaries of ONE addition are
// in registers.  Infinity is tracked in a flag per running sum instead of zz == 0.
template <class F> struct RedSm {
    static constexpr int CH = sizeof(F) / 16, THREADS = 64;
    uint4* base;                                        // [2 sums][4 coordinates][CH chunks][64 threads]
    __device__ __forceinline__ F ld(int acc, int coord) const {
        F v; uint32_t* w = reinterpret_cast<uint32_t*>(&v);
#pragma unroll
        for (int c = 0; c < CH; c++) { uint4 q = base[((acc * 4 + coord) * CH + c) * THREADS]; w[4 * c] = q.x; w[4 * c + 1] = q.y; w[4 * c + 2] = q.z; w[4 * c + 3] = q.w; }
        return v;
    }
    __device__ __forceinline__ void st(int acc, int coord, const F& v) const {
        const uint32_t* w = reinterpret_cast<const uint32_t*>(&v);
#pragma unroll
        for (int c = 0; c < CH; c++) base[((acc * 4 + coord) * CH + c) * THREADS] = make_uint4(w[4 * c], w[4 * c + 1], w[4 * c + 2], w[4 * c + 3]);
    }
};
template <class F> struct RedGlobalOp {                 // addend in global memory
    const XYZZ<F>* p;
    __device__ __forceinline__ bool inf() const { return p->zz.is_zero(); }
    __device__ __forceinline__ F coord(int c) const { return c == 0 ? p->x : (c == 1 ? p->y : (c == 2 ? p->zz : p->zzz)); }
};
template <class F> struct RedSmOp {                     // addend = the other running sum
    RedSm<F> M; int acc; bool is_inf;
    __device__ __forceinline__ bool inf() const { return is_inf; }
    __device__ __forceinline__ F coord(int c) const { return M.ld(acc, c); }
};

template <class F, class Op>
__device__ __forceinline__ void red_sm_add(const RedSm<F>& M, int a, bool& a_inf, const Op& o) {
    if (o.inf()) return;
    if (a_inf) {
#pragma unroll
        for (int c = 0; c < 4; c++) M.st(a, c, o.coord(c));
        a_inf = false;
        return;
    }
    F u1 = M.ld(a, 0) * o.coord(2);
    F p = o.coord(0) * M.ld(a, 2) - u1;
    F s1 = M.ld(a, 1) * o.coord(3);
    F r = o.coord(1) * M.ld(a, 3) - s1;
    if (p.is_zero()) {
        if (r.is_zero()) {                              // equal points: double through registers (rare)
            XYZZ<F> t{M.ld(a, 0), M.ld(a, 1), M.ld(a, 2), M.ld(a, 3)};
            t = t.dbl();
            M.st(a, 0, t.x); M.st(a, 1, t.y); M.st(a, 2, t.zz); M.st(a, 3, t.zzz);
        } else {
            a_inf = true;
        }
        return;
    }
    F pp = p.sqr();
    F ppp = p * pp;
    F q1 = u1 * pp;
    F x3 = r.sqr() - ppp - q1.dbl();
    M.st(a, 0, x3);
    M.st(a, 1, r * (q1 - x3) - s1 * ppp);
    M.st(a, 2, M.ld(a, 2) * o.coord(2) * pp);
    M.st(a, 3, M.ld(a, 3) * o.coord(3) * ppp);
}

template <class F, bool HAS_U>
__global__ void __launch_bounds__(64) k_reduce_level_sm(const XYZZ<F>* __restrict__ S_in, const XYZZ<F>* __restrict__ U_in,
                                                        uint32_t n_in, uint32_t n_out, uint32_t n_groups, uint32_t w_log2,
                                                        uint32_t fan_log2, XYZZ<F>* __restrict__ S_out, XYZZ<F>* __restrict__ U_out) {
    __shared__ uint4 red_sm[2 * 4 * RedSm<F>::CH * 64];
    uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_groups * n_out) return;
    uint32_t g = t / n_out, p = t % n_out;
    const XYZZ<F>* S = S_in + (size_t)g * n_in;
    uint32_t lo = p << fan_log2, hi = min(n_in, lo + (1u << fan_log2));
    RedSm<F> M{red_sm + threadIdx.x};
    bool r_inf = true, t_inf = true;
    for (uint32_t i = hi - 1; i > lo; i--) {
        red_sm_add(M, 0, r_inf, RedGlobalOp<F>{S + i});
        red_sm_add(M, 1, t_inf, RedSmOp<F>{M, 0, r_inf});
    }
    red_sm_add(M, 0, r_inf, RedGlobalOp<F>{S + lo});
    if (w_log2 && !t_inf) {
        XYZZ<F> tt{M.ld(1, 0), M.ld(1, 1), M.ld(1, 2), M.ld(1, 3)};
        for (uint32_t k = 0; k < w_log2; k++) tt = tt.dbl();
        M.st(1, 0, tt.x); M.st(1, 1, tt.y); M.st(1, 2, tt.zz); M.st(1, 3, tt.zzz);
    }
    if (HAS_U) {
        const XYZZ<F>* U = U_in + (size_t)g * n_in;
        for (uint32_t i = lo; i < hi; i++) red_sm_add(M, 1, t_inf, RedGlobalOp<F>{U + i});
    }
    S_out[(size_t)g * n_out + p] = r_inf ? XYZZ<F>::inf() : XYZZ<F>{M.ld(0, 0), M.ld(0, 1), M.ld(0, 2), M.ld(0, 3)};
    U_out[(size_t)g * n_out + p] = t_inf ? XYZZ<F>::inf() : XYZZ<F>{M.ld(1, 0), M.ld(1, 1), M.ld(1, 2), M.ld(1, 3)};
}

// total_g = U_g + S_g   (weights are b+1)
template <class F>
__global__ void __launch_bounds__(64) k_group_total(const XYZZ<F>* __restrict__ S, const XYZZ<F>* __restrict__ U, uint32_t n_groups,
                                                    XYZZ<F>* __restrict__ out) {
    uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= n_groups) return;
    XYZZ<F> a = U[g];
    xyzz_add_ni(&a, &S[g]);
    out[g] = a;
}

// ---- 5b: the reduction above level 0 when there are FEW groups (one-shot MSMs: groups = windows) -------------------------
// Levels 1.. of k_reduce_level then run a few thousand threads that each walk ~23 additions and up to 12 doublings in sequence:
// four such levels are a large share of a one-shot 2^20-point G1 or 2^18-point G2 MSM.  With R_p, T_p the
// level-0 sums of chunk p (2^f buckets each) a group's total is  sum_p (T_p + R_p) + 2^f sum_p p R_p,  and the weighted part
// is taken bit by bit:  sum_p p R_p = sum_k 2^k Q_k,  Q_k = sum of the R_p whose index has bit k set.  The two plain sums and the
// log2(n1) sums Q_k are independent tree reductions (one CTA each: a few strided additions per thread, then log2(threads) levels
// in shared memory); one thread per group finishes with a Horner over the bits.  Depth ~16 + 28 group operations instead of ~120.
constexpr uint32_t TAIL_THREADS = 128, TAIL_SLICE = 512;
#ifndef OG_TAIL_MINB
#define OG_TAIL_MINB 1
#endif
template <class F>
__global__ void __launch_bounds__(TAIL_THREADS, OG_TAIL_MINB) k_tail_sums(const XYZZ<F>* __restrict__ R, const XYZZ<F>* __restrict__ T, uint32_t n1,
                                                            uint32_t n_sums, uint32_t n_slices, XYZZ<F>* __restrict__ out) {
    __shared__ XYZZ<F> a[TAIL_THREADS];
    const uint32_t q = blockIdx.x, g = blockIdx.y, sl = blockIdx.z, tid = threadIdx.x;    // q = 0: sum T, 1: sum R, 2 + k: Q_k
    const XYZZ<F>* src = (q == 0 ? T : R) + (size_t)g * n1;
    XYZZ<F> acc = XYZZ<F>::inf();
    if (q < 2) {
        const uint32_t lo = sl * TAIL_SLICE, hi = min(n1, lo + TAIL_SLICE);
        for (uint32_t p = lo + tid; p < hi; p += TAIL_THREADS) xyzz_add_ni(&acc, &src[p]);
    } else {                                              // the n1 / 2 indices with bit k set, enumerated densely: no idle lanes
        const uint32_t k = q - 2, half = n1 >> 1, lo = sl * (TAIL_SLICE / 2), hi = min(half, lo + TAIL_SLICE / 2);
        for (uint32_t j = lo + tid; j < hi; j += TAIL_THREADS) {
            uint32_t p = ((j >> k) << (k + 1)) | (1u << k) | (j & ((1u << k) - 1));
            xyzz_add_ni(&acc, &src[p]);
        }
    }
    a[tid] = acc;
    __syncthreads();
    for (uint32_t s = TAIL_THREADS / 2; s > 0; s >>= 1) {
        if (tid < s) xyzz_add_ni(&a[tid], &a[tid + s]);
        __syncthreads();
    }
    if (tid == 0) out[((size_t)g * n_sums + q) * n_slices + sl] = a[0];
}

// total_g = sum T + sum R + 2^f * sum_k 2^k Q_k: the slices of every sum are added by a small tree, then one lane walks the
// Horner over the bits (one CTA per group so that the groups sit on different SMs)
template <class F>
__global__ void __launch_bounds__(TAIL_THREADS) k_tail_finish(const XYZZ<F>* __restrict__ partials, uint32_t n_sums, uint32_t n_slices, uint32_t f,
                                                              XYZZ<F>* __restrict__ totals) {
    __shared__ XYZZ<F> a[TAIL_THREADS];
    const uint32_t tid = threadIdx.x, n = n_sums * n_slices;      // <= 128: n_sums <= 16 sums of <= 8 slices
    if (tid < n) a[tid] = partials[(size_t)blockIdx.x * n + tid];
    __syncthreads();
    for (uint32_t s = n_slices / 2; s > 0; s >>= 1) {             // n_slices is a power of two; slice 0 of every sum collects
        if (tid < n && (tid % n_slices) < s) xyzz_add_ni(&a[tid], &a[tid + s]);
        __syncthreads();
    }
    if (tid) return;
    XYZZ<F> v = XYZZ<F>::inf();
    for (int k = (int)n_sums - 3; k >= 0; k--) {
        xyzz_dbl_ni(&v);
        xyzz_add_ni(&v, &a[(2 + k) * n_slices]);
    }
    for (uint32_t i = 0; i < f; i++) xyzz_dbl_ni(&v);
    xyzz_add_ni(&v, &a[0]);
    xyzz_add_ni(&v, &a[n_slices]);
    totals[blockIdx.x] = v;
}

template <class F>
static int32_t msm_buckets(og_ctx* ctx, const Affine<F>* d_table, const uint32_t* d_sorted, const uint32_t* d_offsets,
                           const uint32_t* d_counts, uint32_t n_groups, uint32_t nb, uint64_t n_entries_max, XYZZ<F>* d_buckets,
                           XYZZ<F>* d_lvl, uint32_t* d_heavy, uint32_t* d_perm, XYZZ<F>* d_totals, void* aff_scratch = nullptr,
                           bool few_groups = false) {
    uint32_t n_keys = n_groups * nb;
    constexpr int HT = sizeof(F) == 32 ? 256 : 128;
    OG_CUDA(ctx, cudaMemsetAsync(d_heavy, 0, sizeof(uint32_t), ctx->stream));
    OG_LAUNCHN(ctx, "k_bucket_order", k_bucket_order<F>, n_groups, 1024, 0, d_counts, nb, d_perm);
    // cap: a bucket that would keep one thread busy far longer than the average goes to a whole CTA
    // (skewed scalars: witness 0/1 values, short scalars whose top window has few distinct digits)
    uint64_t avg = n_entries_max / (n_keys ? n_keys : 1);
    uint32_t cap = msm_heavy_cap(avg);
#ifdef OG_EXPERIMENT_AFFINE
    if (aff_scratch) {
        OG_TRY((bucket_acc_affine<F>(ctx, d_table, d_sorted, d_offsets, d_counts, n_keys, cap, avg, d_buckets, d_heavy, d_perm, aff_scratch)));
    } else
#endif
    {
        // the long issue-bound kernel of the MSM: on the lane's low-priority stream when the prover runs chunks in flight
        const char* kn = sizeof(F) == 32 ? "k_bucket_acc_g1" : "k_bucket_acc_g2";
        unsigned grid = (n_keys + 127) / 128;
        cudaStream_t hi = ctx->stream;
        if (ctx->acc_stream) { OG_CUDA(ctx, stream_handoff(ctx->acc_ev, hi, ctx->acc_stream)); ctx->stream = ctx->acc_stream; }
        int32_t rc = [&]() -> int32_t {
#ifdef OG_MSM_G1
            OG_LAUNCHN(ctx, kn, k_bucket_acc_sm1, grid, 128, 0, d_table, d_sorted, d_offsets, d_counts, n_keys, cap, d_buckets, d_heavy, d_perm);
#else
            OG_LAUNCHN(ctx, kn, k_bucket_acc_sm, grid, 128, 0, d_table, d_sorted, d_offsets, d_counts, n_keys, cap, d_buckets, d_heavy, d_perm);
#endif
            return OG_OK;
        }();
        ctx->stream = hi;
        OG_TRY(rc);
        if (ctx->acc_stream) OG_CUDA(ctx, stream_handoff(ctx->acc_ev, ctx->acc_stream, hi));
    }
    {
        // segment sums go to the (still unused) reduction scratch; they fit it while avg < 512 (msm.cuh: msm_heavy_seg)
        uint32_t seg = msm_heavy_seg(avg);
        auto k_heavy = k_bucket_heavy<F, HT>;
        OG_LAUNCHN(ctx, "k_heavy_plan", k_heavy_plan<F>, 1, 256, 0, d_heavy, d_counts, n_keys, seg);
        OG_LAUNCHN(ctx, sizeof(F) == 32 ? "k_bucket_heavy_g1" : "k_bucket_heavy_g2", k_heavy, 4 * ctx->sm_count, HT, HT * sizeof(XYZZ<F>), d_table, d_sorted,
                   d_offsets, d_counts, n_keys, seg, d_lvl, d_heavy);
        OG_LAUNCH(ctx, k_heavy_combine<F>, ctx->sm_count, 32, 0, d_lvl, n_keys, d_buckets, d_heavy);
    }
    // reduction levels
    size_t lvl_stride = (size_t)n_groups * ((nb + RED_FAN - 1) / RED_FAN) + 16;
    XYZZ<F>* bufS[2] = {d_lvl, d_lvl + lvl_stride};
    XYZZ<F>* bufU[2] = {d_lvl + 2 * lvl_stride, d_lvl + 3 * lvl_stride};
    const XYZZ<F>* S_in = d_buckets;
    const XYZZ<F>* U_in = nullptr;
    uint32_t n_in = nb, w_log2 = 0;
    int pp = 0;
    // level 0 (raw buckets) is most of the work: a wider fan there spends fewer additions per bucket (2 - 1/fan)
    // and leaves less for the levels above, at the price of longer serial chains; OG_RED_FAN0 = 3, 4 or 5
    const uint32_t fan0 = [] { const char* v = getenv("OG_RED_FAN0"); int x = v ? atoi(v) : 0; return (uint32_t)(x >= 3 && x <= 5 ? x : RED_FAN_LOG2); }();   // read per call: tests toggle it
    do {
        uint32_t fan_log2 = U_in ? RED_FAN_LOG2 : fan0;
        uint32_t n_out = (n_in + (1u << fan_log2) - 1) >> fan_log2;
        uint32_t threads = n_groups * n_out;
        const char* rn = sizeof(F) == 32 ? "k_reduce_level_g1" : "k_reduce_level_g2";
        // G1: running sums in registers, group operations out of line; G2: running sums in shared memory (the losing
        // combination of each was removed from the library)
        if constexpr (RED_SM_DEFAULT<F>) {
            if (U_in) { auto k = k_reduce_level_sm<F, true>; OG_LAUNCHN(ctx, rn, k, (threads + 63) / 64, 64, 0, S_in, U_in, n_in, n_out, n_groups, w_log2, fan_log2, bufS[pp], bufU[pp]); }
            else { auto k = k_reduce_level_sm<F, false>; OG_LAUNCHN(ctx, rn, k, (threads + 63) / 64, 64, 0, S_in, U_in, n_in, n_out, n_groups, w_log2, fan_log2, bufS[pp], bufU[pp]); }
        } else {
            if (U_in) { auto k = k_reduce_level<F, true>; OG_LAUNCHN(ctx, rn, k, (threads + 63) / 64, 64, 0, S_in, U_in, n_in, n_out, n_groups, w_log2, fan_log2, bufS[pp], bufU[pp]); }
            else { auto k = k_reduce_level<F, false>; OG_LAUNCHN(ctx, rn, k, (threads + 63) / 64, 64, 0, S_in, U_in, n_in, n_out, n_groups, w_log2, fan_log2, bufS[pp], bufU[pp]); }
        }
        S_in = bufS[pp]; U_in = bufU[pp];
        pp ^= 1;
        n_in = n_out;
        w_log2 += fan_log2;
        if (few_groups && w_log2 == fan_log2 && n_in >= 64 && (n_in & (n_in - 1)) == 0) {
            // one-shot MSM: everything above level 0 as independent tree sums + one Horner per group (5b above)
            const bool tail = [] { const char* v = getenv("OG_MSM_TAIL"); return !(v && v[0] == '0' && v[1] == 0); }();   // read per call: tests toggle it
            if (tail) {
                uint32_t n_bits = 0;
                while ((1u << n_bits) < n_in) n_bits++;
                const uint32_t n_sums = n_bits + 2, n_slices = (n_in + TAIL_SLICE - 1) / TAIL_SLICE;
                if (n_sums * n_slices <= TAIL_THREADS) {
                    XYZZ<F>* partials = bufS[pp];                           // the other ping-pong buffer: n_groups * n_in / 8 + 16 >= n_groups * n_sums * n_slices
                    OG_LAUNCHN(ctx, sizeof(F) == 32 ? "k_tail_sums_g1" : "k_tail_sums_g2", k_tail_sums<F>, dim3(n_sums, n_groups, n_slices), TAIL_THREADS, 0,
                               S_in, U_in, n_in, n_sums, n_slices, partials);
                    OG_LAUNCHN(ctx, sizeof(F) == 32 ? "k_tail_finish_g1" : "k_tail_finish_g2", k_tail_finish<F>, n_groups, TAIL_THREADS, 0, partials, n_sums, n_slices,
                               w_log2, d_totals);
                    return OG_OK;
                }
            }
        }
    } while (n_in > 1);
    OG_LAUNCH(ctx, k_group_total<F>, (n_groups + 63) / 64, 64, 0, S_in, U_in, n_groups, d_totals);
    return OG_OK;
}

#ifdef OG_MSM_G1
int32_t msm_buckets_g1(og_ctx* ctx, const G1Affine* d_table, const uint32_t* d_sorted, const uint32_t* d_offsets,
                       const uint32_t* d_counts, uint32_t n_groups, uint32_t nb, uint64_t n_entries_max, G1XYZZ* d_buckets,
                       G1XYZZ* d_lvl, uint32_t* d_heavy, uint32_t* d_perm, G1XYZZ* d_totals, void* aff_scratch) {
    return msm_buckets<Fq>(ctx, d_table, d_sorted, d_offsets, d_counts, n_groups, nb, n_entries_max, d_buckets, d_lvl, d_heavy, d_perm, d_totals, aff_scratch);
}
#ifdef OG_EXPERIMENT_AFFINE
size_t msm_aff_scratch_bytes_g1(uint64_t n_keys) { return aff_scratch_bytes_t<Fq>(n_keys); }
#else
size_t msm_aff_scratch_bytes_g1(uint64_t) { return 0; }
#endif
#endif  // OG_MSM_G1

#ifdef OG_MSM_G2
int32_t msm_buckets_g2(og_ctx* ctx, const G2Affine* d_table, const uint32_t* d_sorted, const uint32_t* d_offsets,
                       const uint32_t* d_counts, uint32_t n_groups, uint32_t nb, uint64_t n_entries_max, G2XYZZ* d_buckets,
                       G2XYZZ* d_lvl, uint32_t* d_heavy, uint32_t* d_perm, G2XYZZ* d_totals, void* aff_scratch) {
    return msm_buckets<Fq2>(ctx, d_table, d_sorted, d_offsets, d_counts, n_groups, nb, n_entries_max, d_buckets, d_lvl, d_heavy, d_perm, d_totals, aff_scratch);
}
#ifdef OG_EXPERIMENT_AFFINE
size_t msm_aff_scratch_bytes_g2(uint64_t n_keys) { return aff_scratch_bytes_t<Fq2>(n_keys); }
#else
size_t msm_aff_scratch_bytes_g2(uint64_t) { return 0; }
#endif
#endif  // OG_MSM_G2

// ---- test/debug probe (og_msm_bucket_sums): msm_buckets on bucket lists the caller gives -------------------------------------
template <class F>
__global__ void __launch_bounds__(128) k_xyzz_to_bytes(const XYZZ<F>* __restrict__ in, uint64_t n, uint8_t* __restrict__ out) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    constexpr int B = FieldIO<F>::BYTES;
    Affine<F> a;
    xyzz_to_affine_ni(&a, &in[i]);
    FieldIO<F>::store(out + 2 * B * i, a.x);
    FieldIO<F>::store(out + 2 * B * i + B, a.y);
}

template <class F>
static int32_t msm_bucket_sums_t(og_ctx* ctx, const uint8_t* d_points, uint32_t n_points, const uint32_t* d_sorted,
                                 const uint32_t* d_offsets, const uint32_t* d_counts, uint32_t n_groups, uint32_t nb,
                                 uint64_t n_entries_max, bool few_groups, uint8_t* d_out_totals, uint8_t* d_out_buckets) {
    const uint32_t n_keys = n_groups * nb;
    OG_SLOT(ctx, pts, Affine<F>, S_MSM_POINTS, sizeof(Affine<F>) * (size_t)n_points);
    OG_SLOT(ctx, buckets, XYZZ<F>, S_MSM_BUCKETS, sizeof(XYZZ<F>) * (size_t)n_keys);
    OG_SLOT(ctx, lvl, XYZZ<F>, S_MSM_SEG, sizeof(XYZZ<F>) * msm_lvl_elems(n_groups, nb));
    OG_SLOT(ctx, heavy, uint32_t, S_MSM_HEAVY, 4 * (2 * (size_t)n_keys + 4));
    OG_SLOT(ctx, perm, uint32_t, S_MSM_CURSOR, 4 * (size_t)n_keys);
    OG_SLOT(ctx, totals, XYZZ<F>, S_MSM_OUT, sizeof(XYZZ<F>) * (size_t)n_groups);
    if (n_points) OG_LAUNCH(ctx, k_points_to_mont<F>, (n_points + 127) / 128, 128, 0, d_points, (uint64_t)n_points, pts, ctx->d_flag);
    OG_TRY((msm_buckets<F>(ctx, pts, d_sorted, d_offsets, d_counts, n_groups, nb, n_entries_max, buckets, lvl, heavy, perm, totals,
                           nullptr, few_groups)));
    OG_LAUNCH(ctx, k_xyzz_to_bytes<F>, (n_groups + 127) / 128, 128, 0, totals, (uint64_t)n_groups, d_out_totals);
    // the buckets as the reduction read them: accumulated, heavy ones combined
    if (d_out_buckets) OG_LAUNCH(ctx, k_xyzz_to_bytes<F>, (n_keys + 127) / 128, 128, 0, buckets, (uint64_t)n_keys, d_out_buckets);
    return OG_OK;
}

#ifdef OG_MSM_G1
int32_t msm_bucket_sums_g1(og_ctx* ctx, const uint8_t* d_points, uint32_t n_points, const uint32_t* d_sorted, const uint32_t* d_offsets,
                           const uint32_t* d_counts, uint32_t n_groups, uint32_t nb, uint64_t n_entries_max, bool few_groups,
                           uint8_t* d_out_totals, uint8_t* d_out_buckets) {
    return msm_bucket_sums_t<Fq>(ctx, d_points, n_points, d_sorted, d_offsets, d_counts, n_groups, nb, n_entries_max, few_groups,
                                 d_out_totals, d_out_buckets);
}
#endif  // OG_MSM_G1

#ifdef OG_MSM_G2
int32_t msm_bucket_sums_g2(og_ctx* ctx, const uint8_t* d_points, uint32_t n_points, const uint32_t* d_sorted, const uint32_t* d_offsets,
                           const uint32_t* d_counts, uint32_t n_groups, uint32_t nb, uint64_t n_entries_max, bool few_groups,
                           uint8_t* d_out_totals, uint8_t* d_out_buckets) {
    return msm_bucket_sums_t<Fq2>(ctx, d_points, n_points, d_sorted, d_offsets, d_counts, n_groups, nb, n_entries_max, few_groups,
                                  d_out_totals, d_out_buckets);
}
#endif  // OG_MSM_G2


// ---- 6: one-shot MSM = Horner over the window totals ------------------------------------------------------
// sum_w 2^(c w) T_w needs c (W - 1) ~ 240 SEQUENTIAL doublings whatever the order, and one thread's multiplier issues a
// product every ~630 cycles, so a single-thread Horner is a visible share of every one-shot MSM.
// The nine products of an XYZZ doubling form three dependency levels of (2, 4, 3) independent products; four warps -- which
// sit on the SM's four schedulers -- take one product each per level and meet at barriers:
//   level 1: v = (2y)^2, xx = x^2     level 2: w = 2y v, s = x v, mm = (3xx)^2, zz' = v zz
//   level 3: m (s - x3), w y, zzz' = w zzz   with x3 = mm - 2s, y3 = m (s - x3) - w y
template <class F>
__global__ void __launch_bounds__(128) k_horner(const XYZZ<F>* __restrict__ totals, uint32_t n_windows, uint32_t c, uint8_t* __restrict__ out) {
    // acc.y is PENDING after a doubling: y = yt - ywy; the warps that need it form it themselves, so a doubling is three
    // barriers (one per dependency level) and no serial epilogue.  Who touches what: x is read in levels 1-2 and rewritten in
    // level 3; zz only by warp 3 (level 2), zzz only by warp 2 (level 3); y is published by warp 0 in level 1.
    __shared__ XYZZ<F> acc;
    __shared__ F l1v, l1xx, l2w, l2s, l2mm, yt, ywy;
    __shared__ int acc_inf;
    const int warp = threadIdx.x >> 5;
    const bool lead = (threadIdx.x & 31) == 0;
    if (threadIdx.x == 0) { acc = XYZZ<F>::inf(); acc_inf = 1; }
    __syncthreads();
    for (int w = (int)n_windows - 1; w >= 0; w--) {
        const int inf_now = acc_inf;                      // every thread reads the flag BEFORE thread 0 may rewrite it below
        __syncthreads();                                  // (racecheck found the missing barrier on the skip path)
        bool ypend = false;
        if (!inf_now) {
            for (uint32_t k = 0; k < c; k++) {
                if (lead) {                               // level 1: v = (2y)^2, xx = x^2
                    if (warp == 0) { F y = ypend ? yt - ywy : acc.y; acc.y = y; F u = y.dbl(); l1v = u.sqr(); }
                    else if (warp == 1) l1xx = acc.x.sqr();
                }
                __syncthreads();
                if (lead) {                               // level 2: w = 2y v, s = x v, mm = (3 xx)^2, zz' = v zz
                    F v = l1v;
                    if (warp == 0) { F u = acc.y.dbl(); l2w = u * v; }
                    else if (warp == 1) l2s = acc.x * v;
                    else if (warp == 2) { F xx = l1xx; F m = xx.dbl() + xx; l2mm = m.sqr(); }
                    else acc.zz = v * acc.zz;
                }
                __syncthreads();
                if (lead) {                               // level 3: m (s - x3), w y, zzz' = w zzz, x3
                    if (warp == 0) { F s = l2s; F x3 = l2mm - s.dbl(); F xx = l1xx; F m = xx.dbl() + xx; yt = m * (s - x3); }
                    else if (warp == 1) ywy = l2w * acc.y;
                    else if (warp == 2) acc.zzz = l2w * acc.zzz;
                    else { F s = l2s; acc.x = l2mm - s.dbl(); }
                }
                __syncthreads();
                ypend = true;
            }
        }
        if (threadIdx.x == 0) {
            XYZZ<F> a = acc;
            if (ypend) a.y = yt - ywy;
            xyzz_add_ni(&a, &totals[w]);
            acc = a;
            acc_inf = a.is_inf() ? 1 : 0;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        XYZZ<F> a = acc;
        Affine<F> r;
        xyzz_to_affine_ni(&r, &a);
        constexpr int B = FieldIO<F>::BYTES;
        FieldIO<F>::store(out, r.x);
        FieldIO<F>::store(out + B, r.y);
    }
}

#ifdef OG_MSM_G1
// GLV front end of the one-shot G1 MSM (glv.cuh): (P_i, k_i) -> (+-P_i, |k1_i|) at index i and (+-phi(P_i), |k2_i|) at index n + i;
// the signs go into the points.  phi(P_i) is MATERIALISED: applying beta at fetch time instead (entries >= n standing for phi of
// point index - n, signs in the scalars) keeps the table at 64 MB but costs a product per phi entry in the accumulation kernel,
// which made the accumulation slower
__global__ void __launch_bounds__(128) k_glv_expand(const uint8_t* __restrict__ scalars, uint64_t n, Fq beta, Affine<Fq>* __restrict__ pts,
                                                    uint32_t* __restrict__ sc2, int* flag) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t* sp = reinterpret_cast<const uint32_t*>(scalars + 32 * i);
    uint32_t k[8], m1[8], m2[8];
#pragma unroll
    for (int j = 0; j < 8; j++) k[j] = sp[j];
    if (!Fr::canonical_lt_mod(k)) {
        atomicOr(flag, 1);
#pragma unroll
        for (int j = 0; j < 8; j++) k[j] = 0;
    }
    bool n1, n2;
    glv_decompose(k, m1, n1, m2, n2);
    Affine<Fq> p = pts[i];
    const Fq yn = p.y.neg();
    Affine<Fq> q{p.x * beta, n2 ? yn : p.y};          // (0, 0) stays (0, 0)
    if (n1) p.y = yn;
    pts[i] = p;
    pts[n + i] = q;
    uint32_t* o1 = sc2 + 8 * i;
    uint32_t* o2 = sc2 + 8 * (n + i);
#pragma unroll
    for (int j = 0; j < 8; j++) { o1[j] = m1[j]; o2[j] = m2[j]; }
}
#endif

static uint32_t pick_window(uint64_t n) {
    uint32_t lg = 0;
    while ((1ull << (lg + 1)) <= n) lg++;
    int c = (int)lg - 3;
    if (c < 2) c = 2;
    if (c > 16) c = 16;
    return (uint32_t)c;
}

template <class F>
static int32_t msm_dev(og_ctx* ctx, const uint8_t* d_points, const uint8_t* d_scalars, uint64_t n, uint8_t* d_out) {
    constexpr int PB = 2 * FieldIO<F>::BYTES;
    if (n >= (1ull << 28)) return OG_E_INVALID;
    if (!aligned32(d_points) || !aligned32(d_scalars)) return OG_E_INVALID;
    if (n == 0) { OG_CUDA(ctx, cudaMemsetAsync(d_out, 0, PB, ctx->stream)); return OG_OK; }
    // G1: GLV halves the scalar length (2n points, 127-bit scalars): same bucket additions, half the windows to reduce and half
    // the sequential doublings of the Horner (OG_GLV=0 switches it off for A/B)
    const bool glv_on = [] { const char* v = getenv("OG_GLV"); return !(v && v[0] == '0' && v[1] == 0); }();   // read per call: tests toggle it
    const bool glv = sizeof(F) == 32 && glv_on && n >= 1024;
    const uint64_t n_in = n;
    if (glv) n = 2 * n;
    uint32_t c = pick_window(n), W = glv ? (128 + c - 1) / c : msm_windows(c), nb = 1u << (c - 1);
    uint32_t n_keys = W * nb;
    OG_SLOT(ctx, pts, Affine<F>, S_MSM_POINTS, sizeof(Affine<F>) * n);
    OG_SLOT(ctx, counts, uint32_t, S_MSM_COUNTS, 4 * (size_t)n_keys);
    OG_SLOT(ctx, offsets, uint32_t, S_MSM_OFFSETS, 4 * ((size_t)n_keys + 1));
    OG_SLOT(ctx, cursor, uint32_t, S_MSM_CURSOR, 4 * (size_t)n_keys);
    OG_SLOT(ctx, sorted, uint32_t, S_MSM_SORTED, 4 * (size_t)n * W);
    OG_SLOT(ctx, buckets, XYZZ<F>, S_MSM_BUCKETS, sizeof(XYZZ<F>) * (size_t)n_keys);
    OG_SLOT(ctx, lvl, XYZZ<F>, S_MSM_SEG, sizeof(XYZZ<F>) * msm_lvl_elems(W, nb));
    OG_SLOT(ctx, heavy, uint32_t, S_MSM_HEAVY, 4 * (2 * (size_t)n_keys + 4));
    OG_SLOT(ctx, totals, XYZZ<F>, S_MSM_OUT, sizeof(XYZZ<F>) * W);
    OG_LAUNCH(ctx, k_points_to_mont<F>, (unsigned)((n_in + 127) / 128), 128, 0, d_points, n_in, pts, ctx->d_flag);
#ifdef OG_MSM_G1
    if (glv) {
        OG_SLOT(ctx, sc2, uint32_t, S_MSM_SCALARS, 32 * (size_t)n);
        uint32_t bl[8];
        for (int i = 0; i < 8; i++) bl[i] = Glv::beta(i);
        const Fq beta = Fq::from_canonical(bl);
        OG_LAUNCH(ctx, k_glv_expand, (unsigned)((n_in + 127) / 128), 128, 0, d_scalars, n_in, beta, reinterpret_cast<Affine<Fq>*>(pts), sc2, ctx->d_flag);
        d_scalars = reinterpret_cast<const uint8_t*>(sc2);
    }
#endif
    DigitPlan plan;
    plan.scalars = reinterpret_cast<const uint32_t*>(d_scalars);
    plan.n = n; plan.scalar_stride = 0; plan.n_problems = 1;
    plan.c = c; plan.n_windows = W; plan.nb = nb;
    plan.key_stride_problem = 0; plan.key_stride_window = 1; plan.tidx_window_stride = 0;
    plan.montgomery = 0;
    OG_TRY(msm_sort_digits(ctx, plan, n_keys, counts, offsets, cursor, sorted));
    void* aff = nullptr;
#ifdef OG_EXPERIMENT_AFFINE
    {   // OG_AFFINE_ONESHOT=1 routes one-shot MSMs through the experiment so that the edge-case tests exercise it
        const char* v = getenv("OG_AFFINE_ONESHOT");
        if (v && atoi(v) > 0) { aff = ctx->slot(S_MSM_AFF, aff_scratch_bytes_t<F>(n_keys)); if (!aff) return OG_E_NOMEM; }
    }
#endif
    OG_TRY((msm_buckets<F>(ctx, pts, sorted, offsets, counts, W, nb, n * W, buckets, lvl, heavy, cursor, totals, aff, true)));
    OG_LAUNCH(ctx, k_horner<F>, 1, 128, 0, totals, W, c, d_out);
    return OG_OK;
}

#ifdef OG_MSM_G1
int32_t msm_g1_dev(og_ctx* ctx, const uint8_t* d_points, const uint8_t* d_scalars, uint64_t n, uint8_t* d_out64) {
    return msm_dev<Fq>(ctx, d_points, d_scalars, n, d_out64);
}
#endif  // OG_MSM_G1

#ifdef OG_MSM_G2
int32_t msm_g2_dev(og_ctx* ctx, const uint8_t* d_points, const uint8_t* d_scalars, uint64_t n, uint8_t* d_out128) {
    return msm_dev<Fq2>(ctx, d_points, d_scalars, n, d_out128);
}
#endif  // OG_MSM_G2


// ---- plain sum of affine points (post all-gather combine in the sharded MSM) ------------------------------------
template <class F, int THREADS>
__global__ void __launch_bounds__(THREADS) k_sum_points(const uint8_t* __restrict__ pts, uint64_t n, uint8_t* __restrict__ out, int* flag) {
    extern __shared__ __align__(32) unsigned char smem_raw[];
    XYZZ<F>* sh = reinterpret_cast<XYZZ<F>*>(smem_raw);
    constexpr int B = FieldIO<F>::BYTES;
    XYZZ<F> acc = XYZZ<F>::inf();
    for (uint64_t i = threadIdx.x; i < n; i += THREADS) {
        const uint8_t* p = pts + 2 * B * i;
        Affine<F> q{FieldIO<F>::load(p, flag), FieldIO<F>::load(p + B, flag)};
        xyzz_madd_ni(&acc, &q);
    }
    sh[threadIdx.x] = acc;
    __syncthreads();
    for (int s = THREADS / 2; s > 0; s >>= 1) {
        if ((int)threadIdx.x < s) xyzz_add_ni(&sh[threadIdx.x], &sh[threadIdx.x + s]);
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        Affine<F> a;
        xyzz_to_affine_ni(&a, &sh[0]);
        FieldIO<F>::store(out, a.x);
        FieldIO<F>::store(out + B, a.y);
    }
}
#ifdef OG_MSM_G1
int32_t sum_g1_dev(og_ctx* ctx, const uint8_t* d_points, uint64_t n, uint8_t* d_out64) {
    auto k = k_sum_points<Fq, 128>;
    OG_LAUNCH(ctx, k, 1, 128, 128 * sizeof(G1XYZZ), d_points, n, d_out64, ctx->d_flag);
    return OG_OK;
}
#endif  // OG_MSM_G1

#ifdef OG_MSM_G2
int32_t sum_g2_dev(og_ctx* ctx, const uint8_t* d_points, uint64_t n, uint8_t* d_out128) {
    auto k = k_sum_points<Fq2, 128>;
    OG_LAUNCH(ctx, k, 1, 128, 128 * sizeof(G2XYZZ), d_points, n, d_out128, ctx->d_flag);
    return OG_OK;
}
#endif  // OG_MSM_G2


// ---- fixed-base window tables ------------------------------------------------------------------------------------
template <class F>
__global__ void __launch_bounds__(64) k_build_table(Affine<F>* __restrict__ table, uint32_t n, uint32_t c, uint32_t n_windows) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Affine<F> p = table[i];
    for (uint32_t w = 1; w < n_windows; w++) {
        XYZZ<F> x = XYZZ<F>::from_affine(p);
        for (uint32_t k = 0; k < c; k++) xyzz_dbl_ni(&x);
        xyzz_to_affine_ni(&p, &x);
        table[(size_t)w * n + i] = p;
    }
}
#ifdef OG_MSM_G1
int32_t msm_build_table_g1(og_ctx* ctx, G1Affine* d_table, uint32_t n, uint32_t c, uint32_t n_windows) {
    if (n) OG_LAUNCH(ctx, k_build_table<Fq>, (n + 63) / 64, 64, 0, d_table, n, c, n_windows);
    return OG_OK;
}
#endif  // OG_MSM_G1

#ifdef OG_MSM_G2
int32_t msm_build_table_g2(og_ctx* ctx, G2Affine* d_table, uint32_t n, uint32_t c, uint32_t n_windows) {
    if (n) OG_LAUNCH(ctx, k_build_table<Fq2>, (n + 63) / 64, 64, 0, d_table, n, c, n_windows);
    return OG_OK;
}
#endif  // OG_MSM_G2


// ---- fixed-base multiplication by the generators (development setup only) ------------------------------------------
// gen_table[w * 255 + d - 1] = d * 2^(8w) * G,  w < 32, d in 1..255
template <class F>
__global__ void __launch_bounds__(32) k_gen_table(Affine<F> gen, Affine<F>* __restrict__ tab) {
    uint32_t w = threadIdx.x;
    if (w >= 32) return;
    XYZZ<F> x = XYZZ<F>::from_affine(gen);
    for (uint32_t k = 0; k < 8 * w; k++) xyzz_dbl_ni(&x);
    Affine<F> base, t;
    xyzz_to_affine_ni(&base, &x);
    XYZZ<F> acc = XYZZ<F>::inf();
    for (uint32_t d = 1; d < 256; d++) {
        xyzz_madd_ni(&acc, &base);
        xyzz_to_affine_ni(&t, &acc);
        tab[w * 255 + d - 1] = t;
    }
}
template <class F>
__global__ void __launch_bounds__(128) k_fixed_mul(const Affine<F>* __restrict__ tab, const uint8_t* __restrict__ scalars, uint64_t n,
                                                   Affine<F>* __restrict__ out, int* flag) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t* sp = reinterpret_cast<const uint32_t*>(scalars + 32 * i);
    uint32_t s[8];
#pragma unroll
    for (int j = 0; j < 8; j++) s[j] = sp[j];
    if (!Fr::canonical_lt_mod(s)) { atomicOr(flag, 1); out[i] = Affine<F>::inf(); return; }
    XYZZ<F> acc = XYZZ<F>::inf();
    for (uint32_t w = 0; w < 32; w++) {
        uint32_t d = (s[w >> 2] >> ((w & 3) * 8)) & 255;
        if (d) xyzz_madd_ni(&acc, &tab[w * 255 + d - 1]);
    }
    Affine<F> r;
    xyzz_to_affine_ni(&r, &acc);
    out[i] = r;
}

#ifdef OG_MSM_G2
static const uint32_t G2_GEN_X0[8] = {0xd992f6edu, 0x46debd5cu, 0xf75edaddu, 0x674322d4u, 0x5e5c4479u, 0x426a0066u, 0x121f1e76u, 0x1800deefu};
static const uint32_t G2_GEN_X1[8] = {0xaef312c2u, 0x97e485b7u, 0x35a9e712u, 0xf1aa4933u, 0x31fb5d25u, 0x7260bfb7u, 0x920d483au, 0x198e9393u};
static const uint32_t G2_GEN_Y0[8] = {0x66fa7daau, 0x4ce6cc01u, 0x0c43d37bu, 0xe3d1e769u, 0x8dcb408fu, 0x4aab7180u, 0xdb8c6debu, 0x12c85ea5u};
static const uint32_t G2_GEN_Y1[8] = {0xd122975bu, 0x55acdadcu, 0x70b38ef3u, 0xbc4b3133u, 0x690c3395u, 0xec9e99adu, 0x585ff075u, 0x090689d0u};
#endif  // OG_MSM_G2


#ifdef OG_MSM_G1
int32_t fixed_base_mul_g1(og_ctx* ctx, const uint8_t* d_scalars, uint64_t n, G1Affine* d_out) {
    if (!ctx->g1_fixed) {
        G1Affine* tab;
        OG_CUDA(ctx, cudaMalloc(&tab, sizeof(G1Affine) * 32 * 255));
        G1Affine gen{Fq::from_u32(1), Fq::from_u32(2)};
        OG_LAUNCH(ctx, k_gen_table<Fq>, 1, 32, 0, gen, tab);
        ctx->g1_fixed = tab;
    }
    if (n) OG_LAUNCH(ctx, k_fixed_mul<Fq>, (unsigned)((n + 127) / 128), 128, 0, (const G1Affine*)ctx->g1_fixed, d_scalars, n, d_out, ctx->d_flag);
    return OG_OK;
}
#endif  // OG_MSM_G1

#ifdef OG_MSM_G2
int32_t fixed_base_mul_g2(og_ctx* ctx, const uint8_t* d_scalars, uint64_t n, G2Affine* d_out) {
    if (!ctx->g2_fixed) {
        G2Affine* tab;
        OG_CUDA(ctx, cudaMalloc(&tab, sizeof(G2Affine) * 32 * 255));
        G2Affine gen{Fq2{Fq::from_canonical(G2_GEN_X0), Fq::from_canonical(G2_GEN_X1)},
                     Fq2{Fq::from_canonical(G2_GEN_Y0), Fq::from_canonical(G2_GEN_Y1)}};
        OG_LAUNCH(ctx, k_gen_table<Fq2>, 1, 32, 0, gen, tab);
        ctx->g2_fixed = tab;
    }
    if (n) OG_LAUNCH(ctx, k_fixed_mul<Fq2>, (unsigned)((n + 127) / 128), 128, 0, (const G2Affine*)ctx->g2_fixed, d_scalars, n, d_out, ctx->d_flag);
    return OG_OK;
}
#endif  // OG_MSM_G2


}  // namespace og
