// owshen_b200/csrc/bjj_impl.cuh -- (included at the end of mimc.cu: it shares the MiMC7 round constants)
// batched BabyJubJub EdDSA-style signature verification on sm_90a.
//
// This is the one kernel whose algorithm the reference defines: it follows
// /root/reference/src/blockchain/tx/owshen_airdrop/babyjubjub/mod.rs --
//   decompress        mod.rs:88-98     verify            mod.rs:99-115
//   projective add    mod.rs:118-140   projective double mod.rs:152-164
//   multiply          mod.rs:68-78     hash (placeholder product)  mod.rs:202-204
// (SURVEY.md section 8f.3).  One thread verifies one signature: two 256-step double-and-add scalar
// multiplications over Fr in the reference's projective coordinates (the one by the fixed BASE through a table of
// 4-bit window multiples built once per context: 64 additions instead of 256 doublings + ~128 additions), compared by cross-multiplication
// instead of two field inversions.  hash_kind = 1 replaces the placeholder product by MultiMiMC7
// (not reference behaviour; the "real hash" variant the survey asks for).
#include "bjj_core.cuh"

namespace og {

__constant__ uint32_t BJJ_BASE_X[8] = {0xbb957051u, 0x2893f3f6u, 0x0534e0b6u, 0x2ab8d801u, 0x9d6277c1u, 0x4eacb2e0u, 0xd63e739bu, 0x0bb77a6au};   // mod.rs:177-183
__constant__ uint32_t BJJ_BASE_Y[8] = {0x872d7d8bu, 0x4b3c257au, 0xb9e13377u, 0xfce0051fu, 0xd16bf9edu, 0x25572e1cu, 0xf7a0b249u, 0x25797203u};

static __device__ __noinline__ Fr mimc7_multi_hash_n(const Fr* in, int n) {     // MultiMiMC7(in[0..n), key 0)
    Fr r = Fr::zero();
    for (int k = 0; k < n; k++) r = r + in[k] + mimc7_hash<false>(in[k], r, nullptr);
    return r;
}
static __device__ __forceinline__ Fr mimc7_multi_hash5(const Fr* in) { return mimc7_multi_hash_n(in, 5); }

// tab[(w * 15 + d - 1) * 2 + {0, 1}] = affine (x, y) of d * 16^w * BASE, w < 64, d in 1..15 (built once per context)
__global__ void __launch_bounds__(64) k_bjj_table(Fr* __restrict__ tab) {
    uint32_t w = threadIdx.x;
    if (w >= 64) return;
    uint32_t bxc[8], byc[8];
#pragma unroll
    for (int k = 0; k < 8; k++) { bxc[k] = BJJ_BASE_X[k]; byc[k] = BJJ_BASE_Y[k]; }
    const Fr A = bjj_a(), D = bjj_d();
    BjjPoint b{Fr::from_canonical(bxc), Fr::from_canonical(byc), Fr::one()};
    for (uint32_t k = 0; k < 4 * w; k++) bjj_double(&b, &A);
    Fr x, y;
    bjj_to_affine(&x, &y, &b);
    BjjPoint base{x, y, Fr::one()}, acc{Fr::zero(), Fr::one(), Fr::zero()};
    for (uint32_t d = 1; d < 16; d++) {
        bjj_add(&acc, &base, &A, &D);
        bjj_to_affine(&x, &y, &acc);
        tab[2 * (w * 15 + d - 1)] = x;
        tab[2 * (w * 15 + d - 1) + 1] = y;
    }
}

static int32_t bjj_table(og_ctx* ctx, const Fr** out) {
    if (!ctx->bjj_fixed) {
        Fr* tab;
        OG_CUDA(ctx, cudaMalloc(&tab, sizeof(Fr) * 2 * 64 * 15));
        OG_LAUNCH(ctx, k_bjj_table, 1, 64, 0, tab);
        ctx->bjj_fixed = tab;
    }
    *out = static_cast<const Fr*>(ctx->bjj_fixed);
    return OG_OK;
}

// out[i]: 1 = verifies, 0 = does not, 2 = the reference would return Err (public key does not decompress)
__global__ void __launch_bounds__(64) k_bjj_verify(const Fr* __restrict__ base_tab, const uint8_t* __restrict__ pk_x, const uint8_t* __restrict__ pk_odd,
                                                   const uint8_t* __restrict__ msgs, const uint8_t* __restrict__ sigs, uint32_t n,
                                                   int hash_kind, uint8_t* __restrict__ out, int* flag) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Fr x = load_canonical<Fr>(pk_x + 32ull * i, flag);
    Fr msg = load_canonical<Fr>(msgs + 32ull * i, flag);
    Fr rx = load_canonical<Fr>(sigs + 96ull * i, flag), ry = load_canonical<Fr>(sigs + 96ull * i + 32, flag);
    Fr s = load_canonical<Fr>(sigs + 96ull * i + 64, flag);
    out[i] = bjj_verify_one(x, pk_odd[i] != 0, msg, rx, ry, s, BjjBase{Fr::zero(), Fr::zero(), base_tab}, [hash_kind](const Fr* in) {
        if (hash_kind == 0) return in[0] * in[1] * in[2] * in[3] * in[4];     // placeholder product, mod.rs:202-204
        return mimc7_multi_hash5(in);
    });
}

// batch of PrivateKey::to_pub + PrivateKey::sign (mod.rs:207-237): one thread per key
__global__ void __launch_bounds__(64) k_bjj_sign(const Fr* __restrict__ base_tab, const uint8_t* __restrict__ sks, const uint8_t* __restrict__ rnds, const uint8_t* __restrict__ msgs,
                                                 uint32_t n, int hash_kind, uint8_t* __restrict__ pk_x, uint8_t* __restrict__ pk_odd,
                                                 uint8_t* __restrict__ sigs, uint8_t* __restrict__ status, int* flag) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Fr sk = load_canonical<Fr>(sks + 32ull * i, flag), rnd = load_canonical<Fr>(rnds + 32ull * i, flag), msg = load_canonical<Fr>(msgs + 32ull * i, flag);
    Fr px, rx, ry, s;
    bool odd;
    uint8_t st = bjj_sign_one(sk, rnd, msg, BjjBase{Fr::zero(), Fr::zero(), base_tab},
        [hash_kind](const Fr* in) { return hash_kind == 0 ? in[0] * in[1] : mimc7_multi_hash_n(in, 2); },
        [hash_kind](const Fr* in) { return hash_kind == 0 ? in[0] * in[1] * in[2] * in[3] * in[4] : mimc7_multi_hash_n(in, 5); },
        &px, &odd, &rx, &ry, &s);
    store_canonical(pk_x + 32ull * i, px);
    pk_odd[i] = odd ? 1 : 0;
    store_canonical(sigs + 96ull * i, rx); store_canonical(sigs + 96ull * i + 32, ry); store_canonical(sigs + 96ull * i + 64, s);
    status[i] = st;
}

int32_t bjj_sign_dev(og_ctx* ctx, const uint8_t* d_sk, const uint8_t* d_rnd, const uint8_t* d_msgs, uint32_t n, int hash_kind,
                     uint8_t* d_pk_x, uint8_t* d_pk_odd, uint8_t* d_sigs, uint8_t* d_status) {
    if (n == 0) return OG_OK;
    const Fr* tab;
    OG_TRY(bjj_table(ctx, &tab));
    OG_LAUNCH(ctx, k_bjj_sign, (n + 63) / 64, 64, 0, tab, d_sk, d_rnd, d_msgs, n, hash_kind, d_pk_x, d_pk_odd, d_sigs, d_status, ctx->d_flag);
    return OG_OK;
}

int32_t bjj_verify_dev(og_ctx* ctx, const uint8_t* d_pk_x, const uint8_t* d_pk_odd, const uint8_t* d_msgs, const uint8_t* d_sigs,
                       uint32_t n, int hash_kind, uint8_t* d_out) {
    if (n == 0) return OG_OK;
    const Fr* tab;
    OG_TRY(bjj_table(ctx, &tab));
    OG_LAUNCH(ctx, k_bjj_verify, (n + 63) / 64, 64, 0, tab, d_pk_x, d_pk_odd, d_msgs, d_sigs, n, hash_kind, d_out, ctx->d_flag);
    return OG_OK;
}

}  // namespace og
