// owshen_b200/csrc/experiments/bucket_acc_g2_smem_operands.cuh -- REJECTED EXPERIMENT, not part of libowshen_b200.so.
// G2 bucket accumulation with EVERY Fq2 value of the mixed addition in shared memory (VERDICT r1 item 4: "pass Fq2 operands to
// the out-of-line multiplier through the shared-memory accumulator layout").  Bit-exact, with far less local-memory traffic per
// addition (128 registers) -- and slower than the shipped kernel, as slow as that kernel at 4 instead of 6 resident CTAs: the
// spills and the marshalling moves are not what bounds the kernel, the multiplier's own instruction mix is (identical in both
// forms).  To repeat: paste into msm.cu inside #ifdef OG_MSM_G2 and
// launch k_bucket_acc_sm2 with 6 * 4 * 128 * 16 bytes of dynamic shared memory instead of k_bucket_acc_sm.
//
//     p   = qx ZZ - X                 -> P        (X is dead after q1, r takes its slot; x3 lands in P and the two
//     pp  = p^2                       -> Q         slots swap roles for the next entry)
//     ZZ  = ZZ pp ;  ppp = p pp       -> P ;  q1 = X pp -> Q
//     r   = qy ZZZ - Y                -> X ;  ZZZ = ZZZ ppp ;  t = Y ppp -> Y
//     x3  = r^2 - ppp - 2 q1          -> P ;  d = q1 - x3 -> Q ;  y3 = r d - t -> Y
#pragma once

__device__ __forceinline__ uint4 lds128(uint32_t a) {
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(a) : "memory");
    return v;
}
__device__ __forceinline__ void sts128(uint32_t a, uint32_t x, uint32_t y, uint32_t z, uint32_t w) {
    asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" :: "r"(a), "r"(x), "r"(y), "r"(z), "r"(w) : "memory");
}
constexpr uint32_t SM2_CHUNK = 128 * 16;          // bytes between the 16-byte chunks of one thread's slot
constexpr uint32_t SM2_SLOT = 4 * SM2_CHUNK;      // bytes between slots

__device__ __forceinline__ void sm2_ld_fq(uint32_t* l, uint32_t a, int half) {
    uint4 u = lds128(a + (2 * half) * SM2_CHUNK), v = lds128(a + (2 * half + 1) * SM2_CHUNK);
    l[0] = u.x; l[1] = u.y; l[2] = u.z; l[3] = u.w; l[4] = v.x; l[5] = v.y; l[6] = v.z; l[7] = v.w;
}
__device__ __forceinline__ Fq2 sm2_ld(uint32_t a) { Fq2 v; sm2_ld_fq(v.c0.l, a, 0); sm2_ld_fq(v.c1.l, a, 1); return v; }
__device__ __forceinline__ void sm2_st(uint32_t a, const Fq2& v) {
    sts128(a, v.c0.l[0], v.c0.l[1], v.c0.l[2], v.c0.l[3]);
    sts128(a + SM2_CHUNK, v.c0.l[4], v.c0.l[5], v.c0.l[6], v.c0.l[7]);
    sts128(a + 2 * SM2_CHUNK, v.c1.l[0], v.c1.l[1], v.c1.l[2], v.c1.l[3]);
    sts128(a + 3 * SM2_CHUNK, v.c1.l[4], v.c1.l[5], v.c1.l[6], v.c1.l[7]);
}
struct SmOperand { uint32_t a; __device__ __forceinline__ void half(uint32_t* l, int h) const { sm2_ld_fq(l, a, h); } };
struct GlobalOperand {                             // an Fq2 of the window table (64 contiguous bytes, read-only)
    const uint4* p;
    __device__ __forceinline__ void half(uint32_t* l, int h) const {
        uint4 u = __ldg(p + 2 * h), v = __ldg(p + 2 * h + 1);
        l[0] = u.x; l[1] = u.y; l[2] = u.z; l[3] = u.w; l[4] = v.x; l[5] = v.y; l[6] = v.z; l[7] = v.w;
    }
};
__device__ __forceinline__ void add8(uint32_t* r, const uint32_t* a, const uint32_t* b) {
    CC cc;
    r[0] = add_cc(a[0], b[0], cc);
#pragma unroll
    for (int j = 1; j < 7; j++) r[j] = addc_cc(a[j], b[j], cc);
    r[7] = addc(a[7], b[7], cc);
}
// Karatsuba with lazy reduction as Fq2::mul_inl, each operand half loaded where the wide product that needs it starts
template <class OA>
__device__ __forceinline__ Fq2 fq2_mul_mem(const OA& A, uint32_t b) {
    uint32_t x[8], y[8], T0[16], T1[16];
    CC cc;
    A.half(x, 0); sm2_ld_fq(y, b, 0); mul_wide(T0, x, y);
    A.half(x, 1); sm2_ld_fq(y, b, 1); mul_wide(T1, x, y);
    Fq2 r;
    {
        uint32_t D[16];                             // c0 = T0 - T1 + p * 2^256
        D[0] = sub_cc(T0[0], T1[0], cc);
#pragma unroll
        for (int j = 1; j < 15; j++) D[j] = subc_cc(T0[j], T1[j], cc);
        D[15] = subc(T0[15], T1[15], cc);
        D[8] = add_cc(D[8], FqParams::mod(0), cc);
#pragma unroll
        for (int j = 1; j < 7; j++) D[8 + j] = addc_cc(D[8 + j], FqParams::mod(j), cc);
        D[15] = addc(D[15], FqParams::mod(7), cc);
        mont_reduce_wide<FqParams>(r.c0.l, D);
        final_sub<FqParams>(r.c0.l);
    }
    T0[0] = add_cc(T0[0], T1[0], cc);               // S = T0 + T1
#pragma unroll
    for (int j = 1; j < 15; j++) T0[j] = addc_cc(T0[j], T1[j], cc);
    T0[15] = addc(T0[15], T1[15], cc);
    {
        uint32_t z[8];                              // c1 = (a0 + a1)(b0 + b1) - S
        A.half(x, 0); A.half(z, 1); add8(x, x, z);
        sm2_ld_fq(y, b, 0); sm2_ld_fq(z, b, 1); add8(y, y, z);
        mul_wide(T1, x, y);
        T1[0] = sub_cc(T1[0], T0[0], cc);
#pragma unroll
        for (int j = 1; j < 15; j++) T1[j] = subc_cc(T1[j], T0[j], cc);
        T1[15] = subc(T1[15], T0[15], cc);
        mont_reduce_wide<FqParams>(r.c1.l, T1);
    }
    return r;
}
static __device__ __noinline__ Fq2 fq2_mul_ss(uint32_t a, uint32_t b) { return fq2_mul_mem(SmOperand{a}, b); }
static __device__ __noinline__ Fq2 fq2_mul_gs(const uint4* a, uint32_t b) { return fq2_mul_mem(GlobalOperand{a}, b); }
static __device__ __noinline__ Fq2 fq2_sqr_s(uint32_t a) {
    Fq a0, a1;
    sm2_ld_fq(a0.l, a, 0); sm2_ld_fq(a1.l, a, 1);
    Fq m = a0 * a1;
    return Fq2{(a0 + a1) * (a0 - a1), m + m};
}

__global__ void __launch_bounds__(128, 4) k_bucket_acc_sm2(const Affine<Fq2>* __restrict__ table, const uint32_t* __restrict__ sorted,
                                                        const uint32_t* __restrict__ offsets, const uint32_t* __restrict__ counts,
                                                        uint32_t n_keys, uint32_t cap, XYZZ<Fq2>* __restrict__ buckets,
                                                        uint32_t* __restrict__ heavy, const uint32_t* __restrict__ perm) {
    extern __shared__ uint4 sm2[];                 // 6 slots x 4 chunks x 128 threads
    uint32_t slot_ = blockIdx.x * blockDim.x + threadIdx.x;
    if (slot_ >= n_keys) return;
    uint32_t key = perm[slot_];
    uint32_t cnt = counts[key], off = offsets[key];
    if (cnt > cap) { uint32_t slot = atomicAdd(heavy, 1u); heavy[1 + slot] = key; buckets[key] = XYZZ<Fq2>::inf(); return; }
    const uint32_t base = (uint32_t)__cvta_generic_to_shared(sm2) + threadIdx.x * 16;
    uint32_t sX = base, sP = base + 4 * SM2_SLOT;   // the two slots that swap roles
    const uint32_t sY = base + SM2_SLOT, sZZ = base + 2 * SM2_SLOT, sZZZ = base + 3 * SM2_SLOT, sQ = base + 5 * SM2_SLOT;
    bool inf = true;
    uint32_t e = cnt ? sorted[off] : 0;
    for (uint32_t k = 0; k < cnt; k++) {
        uint32_t en = k + 1 < cnt ? sorted[off + k + 1] : 0;
        const Affine<Fq2>* tp = table + (e >> 1);
        const bool negq = e & 1;
        e = en;
        const uint4* qx = reinterpret_cast<const uint4*>(&tp->x);
        const uint4* qy = reinterpret_cast<const uint4*>(&tp->y);
        if (inf) {
            Affine<Fq2> q = *tp;
            if (q.is_inf()) continue;
            if (negq) q.y = q.y.neg();
            sm2_st(sX, q.x); sm2_st(sY, q.y); sm2_st(sZZ, Fq2::one()); sm2_st(sZZZ, Fq2::one());
            inf = false;
            continue;
        }
        {
            uint4 o = __ldg(qx);                    // table point at infinity: (0, 0)
#pragma unroll
            for (int c = 1; c < 8; c++) { uint4 v = __ldg(qx + c); o.x |= v.x; o.y |= v.y; o.z |= v.z; o.w |= v.w; }
            if ((o.x | o.y | o.z | o.w) == 0) continue;
        }
        Fq2 p = fq2_mul_gs(qx, sZZ) - sm2_ld(sX);
        if (p.is_zero()) {                          // same x: doubling or cancellation (rare; by-value group code)
            Fq2 s2 = fq2_mul_gs(qy, sZZZ);
            if (negq) s2 = s2.neg();
            Fq2 r = s2 - sm2_ld(sY);
            if (r.is_zero()) {
                Affine<Fq2> q = *tp;
                if (negq) q.y = q.y.neg();
                XYZZ<Fq2> d = XYZZ<Fq2>::dbl_affine(q);
                sm2_st(sX, d.x); sm2_st(sY, d.y); sm2_st(sZZ, d.zz); sm2_st(sZZZ, d.zzz);
            } else inf = true;
            continue;
        }
        sm2_st(sP, p);
        sm2_st(sQ, fq2_sqr_s(sP));                  // pp
        sm2_st(sZZ, fq2_mul_ss(sZZ, sQ));
        sm2_st(sP, fq2_mul_ss(sP, sQ));             // ppp
        sm2_st(sQ, fq2_mul_ss(sX, sQ));             // q1; X is dead from here on
        {
            Fq2 s2 = fq2_mul_gs(qy, sZZZ);
            if (negq) s2 = s2.neg();
            sm2_st(sX, s2 - sm2_ld(sY));            // r
        }
        sm2_st(sZZZ, fq2_mul_ss(sZZZ, sP));
        sm2_st(sY, fq2_mul_ss(sY, sP));             // t = Y ppp
        {
            Fq2 x3 = fq2_sqr_s(sX) - sm2_ld(sP);
            Fq2 q1 = sm2_ld(sQ);
            x3 = x3 - q1.dbl();
            sm2_st(sP, x3);
            sm2_st(sQ, q1 - x3);                    // d
        }
        sm2_st(sY, fq2_mul_ss(sX, sQ) - sm2_ld(sY));
        uint32_t t = sX; sX = sP; sP = t;
    }
    buckets[key] = inf ? XYZZ<Fq2>::inf() : XYZZ<Fq2>{sm2_ld(sX), sm2_ld(sY), sm2_ld(sZZ), sm2_ld(sZZZ)};
}
