// owshen_b200/csrc/experiments/bucket_affine.cuh -- REJECTED EXPERIMENT, not part of libowshen_b200.so.
// Batched-affine bucket accumulation for the prover's MSMs, compared against the XYZZ kernel it was meant to replace:
// bit-exact, but slower once its batched inversion kernels are counted (it moves several hundred bytes of DRAM traffic per
// addition).  Kept so that the measurement can be
// repeated: build msm.cu with -DOG_EXPERIMENT_AFFINE (it is included from there) and run with OG_AFFINE=1 (G1) / 3 (G1 + G2).
#pragma once

// ---- 4b: batched-affine bucket accumulation (the batched prover) ------------------------
// A mixed XYZZ addition costs 8M + 2S; an affine addition costs 1M + 1S + 1M once 1/(x2 - x1) is known, and Montgomery's
// trick turns N inversions into one inversion and 3(N-1) products.  With 10^7 buckets per chunk there are 10^7 independent
// additions available at every step of the bucket lists, so the accumulation runs in ROUNDS: round j adds entry j of every
// bucket list to that bucket's affine accumulator (64 B in HBM).  One kernel per round, k_aff_round:
//   * a thread owns AFF_KB neighbouring buckets of the load-ordered list, a CTA 128 threads;
//   * prologue: the CTA rebuilds the product tree of its threads' denominator products in shared memory and walks it down
//     from 1/(CTA product) -- supplied by the tiny batched inversion over CTA products that runs between rounds
//     (two 32-fold tree levels + Fermat on <= ~1000 values) -- to every thread's own inverse u;
//   * main loop: inv_d = u * pre[slot]; u *= d; lambda, x3, y3; then the denominator of the NEXT round from the fresh
//     accumulator, its running product stored as pre[slot].  The loop direction alternates between rounds so that the
//     exclusive products written by one round are exactly what the next one peels (no second pass, no recomputation);
//   * epilogue: per-thread products -> CTA product.
// Per addition 5M + 1S (+ ~0.3M of trees and inversion) against 8M + 2S; in exchange the accumulator (64 B read + 64 B
// write) and pre (32 B + 32 B) travel through HBM every round -- multiplier time traded for bandwidth the XYZZ kernel
// leaves idle.  Exceptional cases (P + P, P - P, infinity) keep the batch alive by contributing no denominator (or 2y
// for a doubling) and are resolved per slot.  Infinity in the accumulator array is x.l[7] = 0xffffffff (no reduced field
// element looks like that), so a slot is classified from x coordinates alone unless they collide.
constexpr int AFF_KB = 8, AFF_THREADS = 128;
constexpr uint32_t AFF_INF_MARK = 0xffffffffu;

template <class F> struct AffMark;
template <> struct AffMark<Fq> {
    static __device__ __forceinline__ bool is_inf(const Fq& x) { return x.l[7] == AFF_INF_MARK; }
    static __device__ __forceinline__ void set_inf(Fq& x) { x.l[7] = AFF_INF_MARK; }
};
template <> struct AffMark<Fq2> {
    static __device__ __forceinline__ bool is_inf(const Fq2& x) { return x.c0.l[7] == AFF_INF_MARK; }
    static __device__ __forceinline__ void set_inf(Fq2& x) { x.c0.l[7] = AFF_INF_MARK; }
};

enum : int { AFF_SKIP = 0, AFF_SET = 1, AFF_ADD = 2, AFF_DBL = 3, AFF_ZERO = 4 };

// what adding table point `e` does to an accumulator with x = ax, and the denominator d it needs (ADD / DBL only)
template <class F>
__device__ __forceinline__ int aff_classify(const Affine<F>* __restrict__ table, uint32_t e, const F& ax, const Affine<F>* acc_slot, F& px, F& d) {
    const Affine<F>* tp = table + (e >> 1);
    px = tp->x;
    if (px.is_zero() && tp->y.is_zero()) return AFF_SKIP;           // table point at infinity
    if (AffMark<F>::is_inf(ax)) return AFF_SET;
    d = px - ax;
    if (!d.is_zero()) return AFF_ADD;
    F py = tp->y;
    if (e & 1) py = py.neg();
    F ay = acc_slot->y;
    if (py == ay) { d = ay.dbl(); return AFF_DBL; }                   // y != 0 on these curves (odd group order)
    return AFF_ZERO;
}

// slot-ordered (= load-ordered) copies of the list offsets / lengths; buckets above the cap go to k_bucket_heavy
template <class F>
__global__ void __launch_bounds__(128) k_aff_slots(const uint32_t* __restrict__ offsets, const uint32_t* __restrict__ counts, uint32_t n_keys,
                                                   uint32_t cap, const uint32_t* __restrict__ perm, uint32_t* __restrict__ slot_off,
                                                   uint32_t* __restrict__ slot_cnt, uint32_t* __restrict__ heavy, F* __restrict__ cta_tot, uint32_t n_cta) {
    uint32_t slot = blockIdx.x * blockDim.x + threadIdx.x;
    if (slot < n_cta) cta_tot[slot] = F::one();
    if (slot >= n_keys) return;
    uint32_t key = perm[slot];
    uint32_t cnt = counts[key];
    if (cnt > cap) {
        uint32_t h = atomicAdd(heavy, 1u);
        heavy[1 + h] = key;
        cnt = 0;
    }
    slot_off[slot] = offsets[key];
    slot_cnt[slot] = cnt;
}

// shared-memory product tree over the CTA's 128 per-thread values (heap order: node i has children 2i and 2i + 1,
// leaves at 128 .. 255); returns the root in node[1]
template <class F>
__device__ __forceinline__ void aff_tree_up(F* node, const F& leaf) {
    node[AFF_THREADS + threadIdx.x] = leaf;
    for (uint32_t w = AFF_THREADS / 2; w >= 1; w >>= 1) {
        __syncthreads();
        if (threadIdx.x < w) { uint32_t i = w + threadIdx.x; node[i] = node[2 * i] * node[2 * i + 1]; }
    }
    __syncthreads();
}

// round j (FIRST: j = 0 loads entry 0 into the accumulators).  leaves[t]: product of thread t's denominators for THIS
// round on entry, for the next round on exit; cta_inv[c] = 1 / (product over CTA c) for this round; cta_tot[c] receives
// the CTA product for the next round.
template <class F, bool FIRST, int MINB>
__global__ void __launch_bounds__(AFF_THREADS, MINB) k_aff_round(const Affine<F>* __restrict__ table, const uint32_t* __restrict__ sorted,
                                                           const uint32_t* __restrict__ slot_off, const uint32_t* __restrict__ slot_cnt,
                                                           uint32_t n_keys, uint32_t j, Affine<F>* __restrict__ acc, F* __restrict__ pre,
                                                           F* __restrict__ leaves, const F* __restrict__ cta_inv, F* __restrict__ cta_tot) {
    __shared__ F node[2 * AFF_THREADS];
    __shared__ F ninv[2 * AFF_THREADS];
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    // the thread's AFF_KB slots are AFF_THREADS apart: at every step of the loop the CTA touches 128 CONSECUTIVE slots
    // (accumulators, pre, list heads), i.e. fully coalesced 64-byte / 32-byte / 4-byte accesses
    const uint32_t s0 = blockIdx.x * (AFF_KB * AFF_THREADS) + threadIdx.x;
    uint32_t mx = 0;
#pragma unroll
    for (int k = 0; k < AFF_KB; k++) {
        uint32_t c = s0 + k * AFF_THREADS < n_keys ? slot_cnt[s0 + k * AFF_THREADS] : 0;
        mx = c > mx ? c : mx;
    }
    const bool mine = mx > j;
    if (!__syncthreads_or(mine)) return;           // nothing in this CTA this round, hence nothing later: its product stays 1
    F u = F::one();
    if (!FIRST) {
        aff_tree_up(node, mine ? leaves[t] : F::one());
        if (threadIdx.x == 0) ninv[1] = cta_inv[blockIdx.x];
        for (uint32_t w = 2; w <= AFF_THREADS; w <<= 1) {
            __syncthreads();
            if (threadIdx.x < w) { uint32_t i = w + threadIdx.x; ninv[i] = ninv[i >> 1] * node[i ^ 1]; }
        }
        __syncthreads();
        u = ninv[AFF_THREADS + threadIdx.x];
    }
    F run = F::one();
    if (mine) {
#pragma unroll 1
        for (int kk = 0; kk < AFF_KB; kk++) {
            const int k = (j & 1) ? AFF_KB - 1 - kk : kk;
            const uint32_t slot = s0 + k * AFF_THREADS;
            if (slot >= n_keys) continue;
            const uint32_t cnt = slot_cnt[slot];
            if (cnt <= j) continue;
            const uint32_t off = slot_off[slot];
            const uint32_t e = sorted[off + j];
            Affine<F> r;
            bool r_has_y = true;
            if (FIRST) {
                r = fetch_point(table, e);
                if (r.is_inf()) AffMark<F>::set_inf(r.x);
                acc[slot] = r;
            } else {
                F ax = acc[slot].x, px, d;
                int kind = aff_classify(table, e, ax, acc + slot, px, d);
                if (kind == AFF_SKIP) {
                    r.x = ax; r_has_y = false;
                } else if (kind == AFF_SET) {
                    r = fetch_point(table, e);
                    acc[slot] = r;
                } else if (kind == AFF_ZERO) {
                    r = Affine<F>::inf(); AffMark<F>::set_inf(r.x);
                    acc[slot] = r;
                } else {
                    F inv_d = u * pre[slot];
                    u = u * d;
                    F py = table[e >> 1].y;
                    if (e & 1) py = py.neg();
                    F ay = acc[slot].y;
                    F num;
                    if (kind == AFF_ADD) num = py - ay;
                    else { F xx = ax.sqr(); num = xx.dbl() + xx; }
                    F lam = num * inv_d;
                    r.x = lam.sqr() - ax - px;
                    r.y = lam * (ax - r.x) - ay;
                    acc[slot] = r;
                }
            }
            if (cnt > j + 1) {                      // denominator of the next round from the fresh accumulator
                const uint32_t e2 = sorted[off + j + 1];
                F px2, d2;
                Affine<F> rr;
                if (!r_has_y) rr.y = acc[slot].y;
                else rr.y = r.y;
                int k2 = aff_classify(table, e2, r.x, &rr, px2, d2);
                if (k2 == AFF_ADD || k2 == AFF_DBL) { pre[slot] = run; run = run * d2; }
            }
        }
    }
    if (mine) leaves[t] = run;
    aff_tree_up(node, run);
    if (threadIdx.x == 0) cta_tot[blockIdx.x] = node[1];
}

// after the last round: remaining entries (lists longer than the round count) serially in XYZZ, result to key order
template <class F>
__global__ void __launch_bounds__(128) k_aff_finish(const Affine<F>* __restrict__ table, const uint32_t* __restrict__ sorted,
                                                    const uint32_t* __restrict__ slot_off, const uint32_t* __restrict__ slot_cnt,
                                                    const uint32_t* __restrict__ counts, uint32_t n_keys, uint32_t cap, uint32_t rounds,
                                                    const uint32_t* __restrict__ perm, const Affine<F>* __restrict__ acc,
                                                    XYZZ<F>* __restrict__ buckets) {
    uint32_t slot = blockIdx.x * blockDim.x + threadIdx.x;
    if (slot >= n_keys) return;
    uint32_t key = perm[slot];
    if (counts[key] > cap) return;                  // heavy: k_bucket_heavy owns buckets[key]
    uint32_t cnt = slot_cnt[slot], off = slot_off[slot];
    XYZZ<F> r = XYZZ<F>::inf();
    if (cnt) {
        Affine<F> a = acc[slot];
        if (!AffMark<F>::is_inf(a.x)) r = XYZZ<F>{a.x, a.y, F::one(), F::one()};
    }
    for (uint32_t k = rounds; k < cnt; k++) { Affine<F> q = fetch_point(table, sorted[off + k]); xyzz_madd_ni(&r, &q); }
    buckets[key] = r;
}

// ---- batched inversion of n field elements in place: two tree levels of INV_E-fold products, Fermat at the top -------
constexpr uint32_t INV_E = 32;
template <class F>
__global__ void __launch_bounds__(64) k_inv_up(const F* __restrict__ v, uint64_t n, F* __restrict__ prefix, F* __restrict__ group) {
    uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint64_t lo = g * INV_E, hi = lo + INV_E < n ? lo + INV_E : n;
    if (lo >= n) return;
    F p = F::one();
    for (uint64_t i = lo; i < hi; i++) { prefix[i] = p; p = p * v[i]; }
    group[g] = p;
}
template <class F>
__global__ void __launch_bounds__(64) k_inv_down(F* __restrict__ v, uint64_t n, const F* __restrict__ prefix, const F* __restrict__ group_inv) {
    uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint64_t lo = g * INV_E, hi = lo + INV_E < n ? lo + INV_E : n;
    if (lo >= n) return;
    F u = group_inv[g];
    for (uint64_t i = hi; i-- > lo;) { F e = v[i]; v[i] = u * prefix[i]; u = u * e; }
}
template <class F>
__global__ void __launch_bounds__(32) k_inv_fermat(F* __restrict__ v, uint64_t n) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) v[i] = v[i].inv();
}

// scratch (F elements): n prefix + n/E groups + n/E prefix + n/E^2 groups
static inline size_t inv_scratch_elems(uint64_t n) { uint64_t n1 = (n + INV_E - 1) / INV_E, n2 = (n1 + INV_E - 1) / INV_E; return n + 2 * n1 + n2 + 8; }

// out[i] = 1 / v[i]  (v is left untouched only when out != v)
template <class F>
static int32_t batch_invert(og_ctx* ctx, const F* v, F* out, uint64_t n, F* scratch) {
    if (n == 0) return OG_OK;
    uint64_t n1 = (n + INV_E - 1) / INV_E, n2 = (n1 + INV_E - 1) / INV_E;
    F *pre0 = scratch, *g1 = pre0 + n, *pre1 = g1 + n1, *g2 = pre1 + n1;
    if (out != v) OG_CUDA(ctx, cudaMemcpyAsync(out, v, sizeof(F) * n, cudaMemcpyDeviceToDevice, ctx->stream));
    OG_LAUNCHN(ctx, "k_inv_up", k_inv_up<F>, (unsigned)((n1 + 63) / 64), 64, 0, out, n, pre0, g1);
    OG_LAUNCHN(ctx, "k_inv_up", k_inv_up<F>, (unsigned)((n2 + 63) / 64), 64, 0, g1, n1, pre1, g2);
    OG_LAUNCHN(ctx, "k_inv_fermat", k_inv_fermat<F>, (unsigned)((n2 + 31) / 32), 32, 0, g2, n2);
    OG_LAUNCHN(ctx, "k_inv_down", k_inv_down<F>, (unsigned)((n2 + 63) / 64), 64, 0, g1, n1, pre1, g2);
    OG_LAUNCHN(ctx, "k_inv_down", k_inv_down<F>, (unsigned)((n1 + 63) / 64), 64, 0, out, n, pre0, g1);
    return OG_OK;
}

// bytes of scratch msm_buckets needs for the batched-affine accumulation of n_keys buckets
template <class F>
static size_t aff_scratch_bytes_t(uint64_t n_keys) {
    uint64_t n_thr = (n_keys + AFF_KB - 1) / AFF_KB, n_cta = (n_thr + AFF_THREADS - 1) / AFF_THREADS;
    return (sizeof(Affine<F>) + sizeof(F) + 8) * n_keys + sizeof(F) * (n_cta * AFF_THREADS + 2 * n_cta + inv_scratch_elems(n_cta)) + 4096;
}

template <class F>
static int32_t bucket_acc_affine(og_ctx* ctx, const Affine<F>* d_table, const uint32_t* d_sorted, const uint32_t* d_offsets,
                                 const uint32_t* d_counts, uint32_t n_keys, uint32_t cap, uint64_t avg, XYZZ<F>* d_buckets,
                                 uint32_t* d_heavy, const uint32_t* d_perm, void* scratch) {
    const uint32_t n_thr = (n_keys + AFF_KB - 1) / AFF_KB, n_cta = (n_thr + AFF_THREADS - 1) / AFF_THREADS;
    unsigned char* p = static_cast<unsigned char*>(scratch);
    Affine<F>* acc = reinterpret_cast<Affine<F>*>(p); p += sizeof(Affine<F>) * (size_t)n_keys;
    F* pre = reinterpret_cast<F*>(p); p += sizeof(F) * (size_t)n_keys;
    F* leaves = reinterpret_cast<F*>(p); p += sizeof(F) * (size_t)n_cta * AFF_THREADS;
    F* cta_tot = reinterpret_cast<F*>(p); p += sizeof(F) * (size_t)n_cta;
    F* cta_inv = reinterpret_cast<F*>(p); p += sizeof(F) * (size_t)n_cta;
    F* inv_scr = reinterpret_cast<F*>(p); p += sizeof(F) * inv_scratch_elems(n_cta);
    uint32_t* slot_off = reinterpret_cast<uint32_t*>(p); p += 4 * (size_t)n_keys;
    uint32_t* slot_cnt = reinterpret_cast<uint32_t*>(p);
    // rounds: the lists are ~Poisson(avg); beyond avg + 4 sigma + 2 the few remaining entries are cheaper in k_aff_finish
    uint32_t rounds = 0;
    { const char* v = getenv("OG_AFF_ROUNDS"); if (v) rounds = (uint32_t)atoi(v); }
    if (!rounds) { uint32_t sig = 1; while ((uint64_t)sig * sig < avg) sig++; rounds = (uint32_t)avg + 4 * sig + 2; }
    if (rounds > cap) rounds = cap;                 // entries 0 .. rounds-1 of every list are consumed by rounds 0 .. rounds-1
    const bool g1 = sizeof(F) == 32;
    OG_LAUNCHN(ctx, g1 ? "k_aff_slots_g1" : "k_aff_slots_g2", k_aff_slots<F>, (n_keys + 127) / 128, 128, 0, d_offsets, d_counts, n_keys, cap, d_perm,
               slot_off, slot_cnt, d_heavy, cta_tot, n_cta);
    const char* kn = g1 ? "k_bucket_acc_g1" : "k_bucket_acc_g2";
    { auto k0 = k_aff_round<F, true, 1>; OG_LAUNCHN(ctx, kn, k0, n_cta, AFF_THREADS, 0, d_table, d_sorted, slot_off, slot_cnt, n_keys, 0u, acc, pre, leaves, cta_inv, cta_tot); }
    for (uint32_t j = 1; j < rounds; j++) {
        OG_TRY(batch_invert<F>(ctx, cta_tot, cta_inv, n_cta, inv_scr));
        // resident CTAs per SM requested from ptxas (registers <-> warps in flight): measured, OG_AFF_OCC = 5 | 6 | 8
        static const int occ = [] { const char* v = getenv("OG_AFF_OCC"); return v ? atoi(v) : 0; }();
        if (g1 && occ == 6) { auto k1 = k_aff_round<F, false, (sizeof(F) == 32 ? 6 : 2)>; OG_LAUNCHN(ctx, kn, k1, n_cta, AFF_THREADS, 0, d_table, d_sorted, slot_off, slot_cnt, n_keys, j, acc, pre, leaves, cta_inv, cta_tot); }
        else if (g1 && occ == 8) { auto k1 = k_aff_round<F, false, (sizeof(F) == 32 ? 8 : 2)>; OG_LAUNCHN(ctx, kn, k1, n_cta, AFF_THREADS, 0, d_table, d_sorted, slot_off, slot_cnt, n_keys, j, acc, pre, leaves, cta_inv, cta_tot); }
        else { auto k1 = k_aff_round<F, false, (sizeof(F) == 32 ? 5 : 2)>; OG_LAUNCHN(ctx, kn, k1, n_cta, AFF_THREADS, 0, d_table, d_sorted, slot_off, slot_cnt, n_keys, j, acc, pre, leaves, cta_inv, cta_tot); }
    }
    OG_LAUNCHN(ctx, g1 ? "k_aff_finish_g1" : "k_aff_finish_g2", k_aff_finish<F>, (n_keys + 127) / 128, 128, 0, d_table, d_sorted, slot_off, slot_cnt, d_counts,
               n_keys, cap, rounds, d_perm, acc, d_buckets);
    return OG_OK;
}

