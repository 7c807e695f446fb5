// owshen_b200/csrc/ceremony.cu -- the two-phase Groth16 setup ceremony (Bowe-Gabizon-Miers 2017; DESIGN.md section 4b).
// Phase 1 is a powers-of-tau accumulator that contributors update in turn; phase 2 updates one circuit's delta.  Every
// update comes with a record (its public points and Schnorr proofs of knowledge) that anyone can check, and the key is
// sound if one contributor destroyed their secret.  The GPU does the work that grows with the sizes: one scalar
// multiplication per accumulator point (k_scale), inverse NTTs over points for the Lagrange bases (k_intt_level), the
// R1CS column sums of key derivation (k_colsum, heavy columns through the MSM engine) and the random-linear-combination
// MSMs and subgroup checks of verification.  The pairings of verification run on the host (pairing.cu).
#include <algorithm>
#include "groth16.cuh"
#include "host_math.hpp"
#include "msm.cuh"
#include "withdraw_circuit.hpp"

namespace og {

// ---- formats --------------------------------------------------------------------------------------------------------
// OGPT v1: "OGPT" u32 version u32 log_max, tau_g1[2M] alpha_tau_g1[M] beta_tau_g1[M] (64 B), tau_g2[M] beta_g2 (128 B)
// OGPR v1: "OGPR" u32 version, prev_hash[32], then for x in (t, a, b): [x]_1, [x]_2, R = k G1, z = k + c x
// OGDR v1: "OGDR" u32 version, keccak256(pk || vk) of the previous key, [d]_1, [d]_2, R, z
static constexpr uint32_t PT_HDR = 12;
static constexpr uint64_t POK_BYTES = 64 + 128 + 64 + 32;
static constexpr uint64_t PR_BYTES = 8 + 32 + 3 * POK_BYTES;
static constexpr uint64_t DR_BYTES = 8 + 32 + POK_BYTES;
static constexpr uint32_t COL_HEAVY = 512;     // columns with more terms go through the MSM engine
static constexpr uint64_t VK_DELTA2 = 12 + 64 + 128 + 128;

static uint64_t ptau_bytes(uint32_t log_max) { return PT_HDR + (384ull << log_max) + 128; }

struct PtLayout {
    uint32_t log_max;
    uint64_t M, tau1, alpha1, beta1, tau2, beta2;   // byte offsets
};
static bool pt_layout(const uint8_t* b, uint64_t len, PtLayout& L) {
    if (!b || len < PT_HDR || memcmp(b, "OGPT", 4) != 0) return false;
    uint32_t ver, lm;
    memcpy(&ver, b + 4, 4); memcpy(&lm, b + 8, 4);
    if (ver != 1 || lm < 1 || lm > 24 || len != ptau_bytes(lm)) return false;
    L.log_max = lm; L.M = 1ull << lm;
    L.tau1 = PT_HDR; L.alpha1 = L.tau1 + 128 * L.M; L.beta1 = L.alpha1 + 64 * L.M; L.tau2 = L.beta1 + 64 * L.M; L.beta2 = L.tau2 + 128 * L.M;
    return true;
}

// ---- device buffers and secret hygiene -----------------------------------------------------------------------------
struct DevBuf {
    void* p = nullptr;
    ~DevBuf() { if (p) cudaFree(p); }
    template <class T> T* as() const { return reinterpret_cast<T*>(p); }
};
#define OG_ALLOC(ctx, buf, bytes) OG_CUDA(ctx, cudaMalloc(&(buf).p, (bytes) ? (size_t)(bytes) : 32))

static void wipe(void* p, size_t n) { volatile uint8_t* q = reinterpret_cast<volatile uint8_t*>(p); for (size_t i = 0; i < n; i++) q[i] = 0; }

// a 32-byte little-endian hash read as an integer mod r
static Fr fr_from_le_reduce(const uint8_t h[32]) {
    uint8_t be[32];
    for (int i = 0; i < 32; i++) be[i] = h[31 - i];
    return fr_from_be_bytes_reduce(be);
}

// ---- kernels --------------------------------------------------------------------------------------------------------
// k * P with k canonical limbs: one out-of-line body per field
template <class F>
__device__ __noinline__ XYZZ<F> pmul(const Affine<F>& p, const uint32_t* k) { return XYZZ<F>::mul(p, k); }

// out_i = s_i P_i (per_point) or s_0 P_i; s Montgomery
template <class F>
__global__ void __launch_bounds__(128) k_scale(const Affine<F>* __restrict__ in, const Fr* __restrict__ s, uint64_t n, int per_point,
                                               Affine<F>* __restrict__ out) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t k[8];
    s[per_point ? i : 0].to_canonical(k);
    XYZZ<F> r = pmul(in[i], k);
    xyzz_to_affine_ni(&out[i], &r);
}

// out_j = c x^j
__global__ void __launch_bounds__(256) k_powers(Fr c, Fr x, uint64_t n, Fr* __restrict__ out) {
    uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    Fr acc = c, base = x;
    for (uint64_t e = j; e; e >>= 1) {
        if (e & 1) acc = acc * base;
        base = base.sqr();
    }
    out[j] = acc;
}

// sets *bad unless every point is on the curve y^2 = x^3 + b, finite (unless allow_inf) and, for G2, r P = infinity
template <class F>
__global__ void __launch_bounds__(128) k_check_points(const Affine<F>* __restrict__ in, uint64_t n, F b, int allow_inf, int subgroup, int* bad) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Affine<F> p = in[i];
    if (p.is_inf()) { if (!allow_inf) atomicOr(bad, 1); return; }
    if (!(p.y.sqr() == p.x.sqr() * p.x + b)) { atomicOr(bad, 1); return; }
    if (subgroup) {
        uint32_t r[8];
        for (int k = 0; k < 8; k++) r[k] = FrParams::mod(k);
        if (!pmul(p, r).is_inf()) atomicOr(bad, 1);
    }
}

__device__ __forceinline__ uint32_t brev(uint32_t x, uint32_t bits) { return bits ? __brev(x) >> (32 - bits) : 0; }

template <class F>
__global__ void __launch_bounds__(128) k_bitrev_points(const Affine<F>* __restrict__ in, uint32_t log_m, Affine<F>* __restrict__ out) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < (1u << log_m)) out[brev(i, log_m)] = in[i];
}

// one radix-2 decimation-in-time level s (1-based) of the inverse transform, in place on bit-reversed input.
// tw[k] = omega_m^-k (k < m/2); the last level also carries the 1/m (u by 1/m, the twiddle times 1/m).
template <class F>
__global__ void __launch_bounds__(128) k_intt_level(Affine<F>* __restrict__ a, const Fr* __restrict__ tw, uint32_t log_m, uint32_t s, Fr m_inv) {
    uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= (1u << (log_m - 1))) return;
    const uint32_t half = 1u << (s - 1), j = b & (half - 1);
    const uint32_t i0 = ((b >> (s - 1)) << s) | j, i1 = i0 + half;
    const uint32_t e = j << (log_m - s);
    const bool last = s == log_m;
    XYZZ<F> u, v;
    uint32_t k[8];
    if (last) { m_inv.to_canonical(k); u = pmul(a[i0], k); }
    else u = XYZZ<F>::from_affine(a[i0]);
    if (e == 0 && !last) v = XYZZ<F>::from_affine(a[i1]);      // unit twiddle
    else { (last ? tw[e] * m_inv : tw[e]).to_canonical(k); v = pmul(a[i1], k); }
    XYZZ<F> d = v.neg();
    xyzz_add_ni(&d, &u);
    xyzz_add_ni(&u, &v);
    xyzz_to_affine_ni(&a[i0], &u);
    xyzz_to_affine_ni(&a[i1], &d);
}

// out[c] = sum over the column's terms of val * pts[idx] (val canonical); columns above `heavy` terms are left to the MSM engine
template <class F>
__global__ void __launch_bounds__(128) k_colsum(const Affine<F>* __restrict__ pts, const uint32_t* __restrict__ ptr, const uint32_t* __restrict__ idx,
                                                const uint32_t* __restrict__ val, uint32_t n_cols, uint32_t heavy, Affine<F>* __restrict__ out) {
    uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= n_cols) return;
    const uint32_t b = ptr[c], e = ptr[c + 1];
    if (e - b > heavy) return;
    XYZZ<F> acc = XYZZ<F>::inf();
    for (uint32_t t = b; t < e; t++) {
        XYZZ<F> p = pmul(pts[idx[t]], val + 8ull * t);
        xyzz_add_ni(&acc, &p);
    }
    xyzz_to_affine_ni(&out[c], &acc);
}

// out[t] = the boundary bytes of point idx[t]
__global__ void __launch_bounds__(128) k_gather_rows(const uint8_t* __restrict__ src, uint32_t row_bytes, const uint32_t* __restrict__ idx, uint32_t n,
                                                     uint8_t* __restrict__ out) {
    uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t < n) memcpy(out + (uint64_t)row_bytes * t, src + (uint64_t)row_bytes * idx[t], row_bytes);
}

// ---- host helpers around the kernels --------------------------------------------------------------------------------
static unsigned blocks(uint64_t n, unsigned t) { return (unsigned)((n + t - 1) / t); }

template <class F> static F curve_b() {
    if constexpr (sizeof(F) == sizeof(Fq)) return Fq::from_u32(3);
    else return Fq2{Fq::from_u32(3), Fq::zero()} * Fq2{Fq::from_u32(9), Fq::from_u32(1)}.inv();
}

static int32_t powers(og_ctx* ctx, const Fr& c, const Fr& x, uint64_t n, Fr* d_out) {
    if (n) OG_LAUNCH(ctx, k_powers, blocks(n, 256), 256, 0, c, x, n, d_out);
    return OG_OK;
}

template <class F>
static int32_t scale(og_ctx* ctx, const Affine<F>* d_in, const Fr* d_s, uint64_t n, int per_point, Affine<F>* d_out) {
    if (n) OG_LAUNCH(ctx, k_scale<F>, blocks(n, 128), 128, 0, d_in, d_s, n, per_point, d_out);
    return OG_OK;
}

// in place on 2^log_m affine Montgomery points: [P_j] -> [(1/m) sum_k omega^-jk P_k]
template <class F>
static int32_t intt(og_ctx* ctx, Affine<F>* d, uint32_t log_m) {
    if (log_m == 0) return OG_OK;
    const uint64_t m = 1ull << log_m;
    DevBuf tmp, tw;
    OG_ALLOC(ctx, tmp, sizeof(Affine<F>) * m);
    OG_ALLOC(ctx, tw, sizeof(Fr) * (m / 2));
    OG_TRY(powers(ctx, Fr::one(), host_root_of_unity(log_m).inv(), m / 2, tw.as<Fr>()));
    OG_CUDA(ctx, cudaMemcpyAsync(tmp.p, d, sizeof(Affine<F>) * m, cudaMemcpyDeviceToDevice, ctx->stream));
    OG_LAUNCH(ctx, k_bitrev_points<F>, blocks(m, 128), 128, 0, tmp.as<Affine<F>>(), log_m, d);
    const Fr m_inv = Fr::from_u32(1u << log_m).inv();
    for (uint32_t s = 1; s <= log_m; s++) OG_LAUNCH(ctx, k_intt_level<F>, blocks(m / 2, 128), 128, 0, d, tw.as<Fr>(), log_m, s, m_inv);
    OG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return OG_OK;
}

// boundary bytes in, boundary bytes out: out_i = s P_i for one host scalar
template <class F>
static int32_t scale_bytes_host(og_ctx* ctx, const uint8_t* in, uint64_t n, const Fr& s, uint8_t* out) {
    const uint64_t PB = sizeof(Affine<F>);
    DevBuf db, dm, ds;
    OG_ALLOC(ctx, db, PB * n); OG_ALLOC(ctx, dm, PB * n); OG_ALLOC(ctx, ds, sizeof(Fr));
    OG_CUDA(ctx, cudaMemcpyAsync(db.p, in, PB * n, cudaMemcpyHostToDevice, ctx->stream));
    OG_CUDA(ctx, cudaMemcpyAsync(ds.p, &s, sizeof(Fr), cudaMemcpyHostToDevice, ctx->stream));
    OG_TRY(points_bytes_to_mont(ctx, db.as<uint8_t>(), n, dm.as<Affine<F>>()));
    OG_TRY(scale<F>(ctx, dm.as<Affine<F>>(), ds.as<Fr>(), n, 0, dm.as<Affine<F>>()));
    OG_TRY(points_mont_to_bytes(ctx, dm.as<Affine<F>>(), n, db.as<uint8_t>()));
    OG_CUDA(ctx, cudaMemcpyAsync(out, db.p, PB * n, cudaMemcpyDeviceToHost, ctx->stream));
    OG_CUDA(ctx, cudaMemsetAsync(ds.p, 0, sizeof(Fr), ctx->stream));
    return check_flag(ctx);
}

// x G1 and x G2 for host scalars (canonical bytes out)
static int32_t gen_mul(og_ctx* ctx, const Fr* xs, int n, uint8_t* g1_out, uint8_t* g2_out) {
    DevBuf ds, dp, db;
    OG_ALLOC(ctx, ds, 32 * n); OG_ALLOC(ctx, dp, sizeof(G2Affine) * n); OG_ALLOC(ctx, db, 128 * n);
    std::vector<uint8_t> s(32 * n);
    for (int i = 0; i < n; i++) host_store(s.data() + 32 * i, xs[i]);
    OG_CUDA(ctx, cudaMemcpyAsync(ds.p, s.data(), 32 * n, cudaMemcpyHostToDevice, ctx->stream));
    OG_TRY(fixed_base_mul(ctx, ds.as<uint8_t>(), n, dp.as<G1Affine>()));
    OG_TRY(points_mont_to_bytes(ctx, dp.as<G1Affine>(), n, db.as<uint8_t>()));
    OG_CUDA(ctx, cudaMemcpyAsync(g1_out, db.p, 64 * n, cudaMemcpyDeviceToHost, ctx->stream));
    OG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (g2_out) {
        OG_TRY(fixed_base_mul(ctx, ds.as<uint8_t>(), n, dp.as<G2Affine>()));
        OG_TRY(points_mont_to_bytes(ctx, dp.as<G2Affine>(), n, db.as<uint8_t>()));
        OG_CUDA(ctx, cudaMemcpyAsync(g2_out, db.p, 128 * n, cudaMemcpyDeviceToHost, ctx->stream));
    }
    OG_CUDA(ctx, cudaMemsetAsync(ds.p, 0, 32 * n, ctx->stream));
    OG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    wipe(s.data(), s.size());
    return OG_OK;
}

static int32_t generators(og_ctx* ctx, uint8_t g1[64], uint8_t g2[128]) {
    Fr one = Fr::one();
    return gen_mul(ctx, &one, 1, g1, g2);
}

// ---- proofs of knowledge --------------------------------------------------------------------------------------------
static Fr pok_challenge(const uint8_t prev_hash[32], uint32_t index, const uint8_t* x1, const uint8_t* x2, const uint8_t* R) {
    std::vector<uint8_t> m;
    const char* tag = "OG-ceremony-pok";
    m.insert(m.end(), tag, tag + strlen(tag));
    m.insert(m.end(), prev_hash, prev_hash + 32);
    for (int i = 0; i < 4; i++) m.push_back((uint8_t)(index >> (8 * i)));
    m.insert(m.end(), x1, x1 + 64); m.insert(m.end(), x2, x2 + 128); m.insert(m.end(), R, R + 64);
    uint8_t h[32];
    keccak256(m.data(), m.size(), h);
    return fr_from_le_reduce(h);
}

// writes [x]_1, [x]_2, R, z for each secret (record layout), nonces k
static int32_t make_poks(og_ctx* ctx, const uint8_t prev_hash[32], const Fr* x, const Fr* k, int n, uint8_t* out) {
    std::vector<uint8_t> X1(64 * n), X2(128 * n), R1(64 * n);
    OG_TRY(gen_mul(ctx, x, n, X1.data(), X2.data()));
    OG_TRY(gen_mul(ctx, k, n, R1.data(), nullptr));
    for (int i = 0; i < n; i++) {
        uint8_t* o = out + POK_BYTES * i;
        memcpy(o, &X1[64 * i], 64); memcpy(o + 64, &X2[128 * i], 128); memcpy(o + 192, &R1[64 * i], 64);
        Fr c = pok_challenge(prev_hash, (uint32_t)i, o, o + 64, o + 192);
        Fr z = k[i] + c * x[i];
        host_store(o + 256, z);
        wipe(&z, sizeof(z));
    }
    return OG_OK;
}

// a record entry: points on the curve and finite, z G1 == R + c [x]_1, e([x]_1, G2) == e(G1, [x]_2); X1/X2 out
static bool check_pok(const uint8_t prev_hash[32], uint32_t index, const uint8_t* e, const G1Affine& g1, const G2Affine& g2, G1Affine& X1,
                      G2Affine& X2) {
    G1Affine R;
    Fr z;
    if (!load_g1(X1, e) || !load_g2(X2, e + 64) || !load_g1(R, e + 192) || !host_load(z, e + 256)) return false;
    if (X1.is_inf() || X2.is_inf() || R.is_inf()) return false;
    Fr c = pok_challenge(prev_hash, index, e, e + 64, e + 192);
    uint32_t zk[8], ck[8];
    z.to_canonical(zk); c.to_canonical(ck);
    G1XYZZ lhs = G1XYZZ::mul(g1, zk), rhs = G1XYZZ::mul(X1, ck);
    rhs.madd(R);
    if (!(lhs.to_affine() == rhs.to_affine())) return false;
    const G1Affine P[2] = {X1, g1.neg()};
    const G2Affine Q[2] = {g2, X2};
    return pairing_product_is_one(P, Q, 2);
}

// e(P0, Q0) == e(P1, Q1)
static bool pair_eq(const G1Affine& P0, const G2Affine& Q0, const G1Affine& P1, const G2Affine& Q1) {
    const G1Affine P[2] = {P0, P1.neg()};
    const G2Affine Q[2] = {Q0, Q1};
    return pairing_product_is_one(P, Q, 2);
}

// Fiat-Shamir challenge of a verification: rho = keccak256(tag || H(prev) || H(next) || H(record)) mod r
static Fr fs_rho(const uint8_t* prev, uint64_t prev_len, const uint8_t* next, uint64_t next_len, const uint8_t* rec, uint64_t rec_len) {
    std::vector<uint8_t> m;
    const char* tag = "OG-ceremony-rho";
    m.insert(m.end(), tag, tag + strlen(tag));
    uint8_t h[32];
    keccak256(prev, prev_len, h); m.insert(m.end(), h, h + 32);
    keccak256(next, next_len, h); m.insert(m.end(), h, h + 32);
    keccak256(rec, rec_len, h); m.insert(m.end(), h, h + 32);
    keccak256(m.data(), m.size(), h);
    return fr_from_le_reduce(h);
}

// S0 = sum_{i < n-1} rho^i P_i and S1 = sum_{i < n-1} rho^i P_{i+1} of n consecutive boundary-byte points on the device
template <class F>
static int32_t shifted_sums(og_ctx* ctx, const uint8_t* d_pts, uint64_t n, const uint8_t* d_rho, uint8_t* s0, uint8_t* s1) {
    const uint64_t PB = sizeof(Affine<F>);
    DevBuf out;
    OG_ALLOC(ctx, out, 2 * PB);
    OG_TRY(msm_dev<F>(ctx, d_pts, d_rho, n - 1, out.as<uint8_t>()));
    OG_TRY(msm_dev<F>(ctx, d_pts + PB, d_rho, n - 1, out.as<uint8_t>() + PB));
    OG_CUDA(ctx, cudaMemcpyAsync(s0, out.p, PB, cudaMemcpyDeviceToHost, ctx->stream));
    OG_CUDA(ctx, cudaMemcpyAsync(s1, out.as<uint8_t>() + PB, PB, cudaMemcpyDeviceToHost, ctx->stream));
    OG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return OG_OK;
}

// rho^i, i < n, as canonical bytes on the device
static int32_t rho_powers(og_ctx* ctx, const Fr& rho, uint64_t n, DevBuf& out) {
    DevBuf m;
    OG_ALLOC(ctx, m, sizeof(Fr) * n);
    OG_ALLOC(ctx, out, 32 * n);
    OG_TRY(powers(ctx, Fr::one(), rho, n, m.as<Fr>()));
    OG_TRY(mimc_from_mont_dev(ctx, m.as<Fr>(), n, out.as<uint8_t>()));
    OG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return OG_OK;
}

// every point of d_bytes[n] on the curve, in the subgroup and (unless allow_inf) finite
template <class F>
static int32_t check_points(og_ctx* ctx, const uint8_t* d_bytes, uint64_t n, int allow_inf, bool* ok) {
    DevBuf dm, bad;
    OG_ALLOC(ctx, dm, sizeof(Affine<F>) * n);
    OG_ALLOC(ctx, bad, sizeof(int));
    OG_CUDA(ctx, cudaMemsetAsync(bad.p, 0, sizeof(int), ctx->stream));
    OG_TRY(clear_flag(ctx));
    OG_TRY(points_bytes_to_mont(ctx, d_bytes, n, dm.as<Affine<F>>()));
    const int subgroup = sizeof(F) != sizeof(Fq);
    if (n) OG_LAUNCH(ctx, k_check_points<F>, blocks(n, 128), 128, 0, dm.as<Affine<F>>(), n, curve_b<F>(), allow_inf, subgroup, bad.as<int>());
    int h = 0;
    OG_CUDA(ctx, cudaMemcpyAsync(&h, bad.p, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    OG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    int32_t rc = check_flag(ctx);                  // a non-canonical coordinate
    *ok = rc == OG_OK && h == 0;
    return rc == OG_E_ENCODING ? OG_OK : rc;
}

// ---- phase 1 --------------------------------------------------------------------------------------------------------
int32_t ptau_new(og_ctx* ctx, uint32_t log_max, uint8_t* out, uint64_t* out_len) {
    if (!out_len || log_max < 1 || log_max > 24) return OG_E_INVALID;
    const uint64_t need = ptau_bytes(log_max), M = 1ull << log_max;
    if (!out) { *out_len = need; return OG_OK; }
    if (*out_len < need) return OG_E_INVALID;
    uint8_t g1[64], g2[128];
    OG_TRY(generators(ctx, g1, g2));
    memcpy(out, "OGPT", 4);
    const uint32_t hdr[2] = {1, log_max};
    memcpy(out + 4, hdr, 8);
    uint8_t* p = out + PT_HDR;
    for (uint64_t i = 0; i < 4 * M; i++, p += 64) memcpy(p, g1, 64);
    for (uint64_t i = 0; i < M + 1; i++, p += 128) memcpy(p, g2, 128);
    *out_len = need;
    return OG_OK;
}

int32_t ptau_contribute(og_ctx* ctx, const uint8_t* acc, uint64_t acc_len, const uint8_t* secrets96, const uint8_t* nonces96,
                        uint8_t* acc_out, uint64_t* acc_out_len, uint8_t* rec_out, uint64_t* rec_len) {
    PtLayout L;
    if (!acc_out_len || !rec_len || !pt_layout(acc, acc_len, L)) return OG_E_INVALID;
    if (!acc_out || !rec_out) { *acc_out_len = acc_len; *rec_len = PR_BYTES; return OG_OK; }
    if (*acc_out_len < acc_len || *rec_len < PR_BYTES || !secrets96 || !nonces96) return OG_E_INVALID;
    Fr x[3], k[3];
    int32_t rc = OG_OK;
    for (int i = 0; i < 3; i++)
        if (!host_load(x[i], secrets96 + 32 * i) || !host_load(k[i], nonces96 + 32 * i)) rc = OG_E_ENCODING;
    for (int i = 0; rc == OG_OK && i < 3; i++) if (x[i].is_zero() || k[i].is_zero()) rc = OG_E_INVALID;
    if (rc == OG_OK) {
        rc = [&]() -> int32_t {
            const uint64_t M = L.M, n1 = 4 * M, n2 = M + 1;
            DevBuf db, d1, d2, s1, s2;
            OG_ALLOC(ctx, db, acc_len); OG_ALLOC(ctx, d1, sizeof(G1Affine) * n1); OG_ALLOC(ctx, d2, sizeof(G2Affine) * n2);
            OG_ALLOC(ctx, s1, sizeof(Fr) * n1); OG_ALLOC(ctx, s2, sizeof(Fr) * n2);
            OG_TRY(clear_flag(ctx));
            OG_CUDA(ctx, cudaMemcpyAsync(db.p, acc, acc_len, cudaMemcpyHostToDevice, ctx->stream));
            OG_TRY(points_bytes_to_mont(ctx, db.as<uint8_t>() + L.tau1, n1, d1.as<G1Affine>()));
            OG_TRY(points_bytes_to_mont(ctx, db.as<uint8_t>() + L.tau2, n2, d2.as<G2Affine>()));
            // G1 scalars: t^i (2M), a t^i (M), b t^i (M); G2 scalars: t^i (M), b
            Fr* S1 = s1.as<Fr>(); Fr* S2 = s2.as<Fr>();
            OG_TRY(powers(ctx, Fr::one(), x[0], 2 * M, S1));
            OG_TRY(powers(ctx, x[1], x[0], M, S1 + 2 * M));
            OG_TRY(powers(ctx, x[2], x[0], M, S1 + 3 * M));
            OG_TRY(powers(ctx, Fr::one(), x[0], M, S2));
            OG_TRY(powers(ctx, x[2], x[0], 1, S2 + M));
            OG_TRY(scale<Fq>(ctx, d1.as<G1Affine>(), S1, n1, 1, d1.as<G1Affine>()));
            OG_TRY(scale<Fq2>(ctx, d2.as<G2Affine>(), S2, n2, 1, d2.as<G2Affine>()));
            OG_CUDA(ctx, cudaMemsetAsync(s1.p, 0, sizeof(Fr) * n1, ctx->stream));
            OG_CUDA(ctx, cudaMemsetAsync(s2.p, 0, sizeof(Fr) * n2, ctx->stream));
            OG_TRY(points_mont_to_bytes(ctx, d1.as<G1Affine>(), n1, db.as<uint8_t>() + L.tau1));
            OG_TRY(points_mont_to_bytes(ctx, d2.as<G2Affine>(), n2, db.as<uint8_t>() + L.tau2));
            OG_CUDA(ctx, cudaMemcpyAsync(acc_out + PT_HDR, db.as<uint8_t>() + PT_HDR, acc_len - PT_HDR, cudaMemcpyDeviceToHost, ctx->stream));
            OG_TRY(check_flag(ctx));
            memcpy(acc_out, acc, PT_HDR);
            memcpy(rec_out, "OGPR", 4);
            const uint32_t ver = 1;
            memcpy(rec_out + 4, &ver, 4);
            keccak256(acc, acc_len, rec_out + 8);
            return make_poks(ctx, rec_out + 8, x, k, 3, rec_out + 40);
        }();
    }
    wipe(x, sizeof(x)); wipe(k, sizeof(k));
    if (rc == OG_OK) { *acc_out_len = acc_len; *rec_len = PR_BYTES; }
    return rc;
}

int32_t ptau_verify(og_ctx* ctx, const uint8_t* prev, uint64_t prev_len, const uint8_t* next, uint64_t next_len, const uint8_t* rec,
                    uint64_t rec_len) {
    PtLayout L, L0;
    if (!pt_layout(prev, prev_len, L0) || !pt_layout(next, next_len, L) || L.log_max != L0.log_max) return OG_E_VERIFY;
    if (!rec || rec_len != PR_BYTES || memcmp(rec, "OGPR", 4) != 0) return OG_E_VERIFY;
    uint32_t ver;
    memcpy(&ver, rec + 4, 4);
    uint8_t h[32];
    keccak256(prev, prev_len, h);
    if (ver != 1 || memcmp(h, rec + 8, 32) != 0) return OG_E_VERIFY;
    uint8_t g1b[64], g2b[128];
    OG_TRY(generators(ctx, g1b, g2b));
    if (memcmp(next + L.tau1, g1b, 64) != 0 || memcmp(next + L.tau2, g2b, 128) != 0) return OG_E_VERIFY;
    G1Affine g1; G2Affine g2;
    load_g1(g1, g1b); load_g2(g2, g2b);
    // the record: proofs of knowledge of t, a, b
    G1Affine X1[3]; G2Affine X2[3];
    for (uint32_t i = 0; i < 3; i++)
        if (!check_pok(rec + 8, i, rec + 40 + POK_BYTES * i, g1, g2, X1[i], X2[i])) return OG_E_VERIFY;
    // every point of the new accumulator on the curve and finite, G2 in the subgroup
    const uint64_t M = L.M;
    DevBuf db;                                     // the points without the header: the MSM engine takes 32-byte aligned input
    OG_ALLOC(ctx, db, next_len - PT_HDR);
    OG_CUDA(ctx, cudaMemcpyAsync(db.p, next + PT_HDR, next_len - PT_HDR, cudaMemcpyHostToDevice, ctx->stream));
    const uint8_t* d = db.as<uint8_t>() - PT_HDR;  // indexed by blob offsets
    bool ok1, ok2;
    OG_TRY(check_points<Fq>(ctx, d + L.tau1, 4 * M, 0, &ok1));
    OG_TRY(check_points<Fq2>(ctx, d + L.tau2, M + 1, 0, &ok2));
    if (!ok1 || !ok2) return OG_E_VERIFY;
    // the update: new / old = t, a, b
    G1Affine nt1, na0, nb0, ot1, oa0, ob0;
    G2Affine nt2, nbeta2;
    if (!load_g1(nt1, next + L.tau1 + 64) || !load_g1(na0, next + L.alpha1) || !load_g1(nb0, next + L.beta1) ||
        !load_g1(ot1, prev + L.tau1 + 64) || !load_g1(oa0, prev + L.alpha1) || !load_g1(ob0, prev + L.beta1) ||
        !load_g2(nt2, next + L.tau2 + 128) || !load_g2(nbeta2, next + L.beta2)) return OG_E_VERIFY;
    if (!pair_eq(nt1, g2, ot1, X2[0]) || !pair_eq(na0, g2, oa0, X2[1]) || !pair_eq(nb0, g2, ob0, X2[2]) || !pair_eq(nb0, g2, g1, nbeta2))
        return OG_E_VERIFY;
    // each sequence geometric with ratio tau, batched with the powers of rho
    DevBuf rho;
    OG_TRY(rho_powers(ctx, fs_rho(prev, prev_len, next, next_len, rec, rec_len), 2 * M, rho));
    const struct { uint64_t off, n; } seq1[3] = {{L.tau1, 2 * M}, {L.alpha1, M}, {L.beta1, M}};
    for (auto& s : seq1) {
        uint8_t b0[64], b1[64];
        OG_TRY(shifted_sums<Fq>(ctx, d + s.off, s.n, rho.as<uint8_t>(), b0, b1));
        G1Affine S0, S1;
        if (!load_g1(S0, b0) || !load_g1(S1, b1) || !pair_eq(S1, g2, S0, nt2)) return OG_E_VERIFY;
    }
    uint8_t c0[128], c1[128];
    OG_TRY(shifted_sums<Fq2>(ctx, d + L.tau2, M, rho.as<uint8_t>(), c0, c1));
    G2Affine T0, T1;
    if (!load_g2(T0, c0) || !load_g2(T1, c1) || !pair_eq(g1, T1, nt1, T0)) return OG_E_VERIFY;
    return OG_OK;
}

// ---- key derivation -------------------------------------------------------------------------------------------------
// columns of a sparse matrix: terms ptr[c] .. ptr[c+1] are (point index, canonical coefficient)
struct Cols {
    std::vector<uint32_t> ptr, idx, val;
};
struct Term { uint32_t col, pt; Fr v; };
static void csr_terms(const Csr& M, uint32_t pt_offset, std::vector<Term>& out) {
    for (uint32_t j = 0; j + 1 < M.row_ptr.size(); j++)
        for (uint32_t k = M.row_ptr[j]; k < M.row_ptr[j + 1]; k++) out.push_back({M.col[k], pt_offset + j, M.val[k]});
}
static Cols transpose(uint32_t n_cols, const std::vector<Term>& t) {
    Cols c;
    c.ptr.assign(n_cols + 1, 0);
    for (auto& x : t) c.ptr[x.col + 1]++;
    for (uint32_t i = 0; i < n_cols; i++) c.ptr[i + 1] += c.ptr[i];
    c.idx.resize(t.size()); c.val.resize(8 * t.size());
    std::vector<uint32_t> cur(c.ptr.begin(), c.ptr.end() - 1);
    for (auto& x : t) { uint32_t k = cur[x.col]++; c.idx[k] = x.pt; host_store(reinterpret_cast<uint8_t*>(&c.val[8ull * k]), x.v); }
    return c;
}

// out_host[c] = sum over column c of coefficient * point (boundary bytes); d_pts Montgomery, d_pts_bytes the same points as bytes
template <class F>
static int32_t column_sums(og_ctx* ctx, const Affine<F>* d_pts, const uint8_t* d_pts_bytes, const Cols& c, uint8_t* out_host) {
    const uint64_t PB = sizeof(Affine<F>);
    const uint32_t n_cols = (uint32_t)c.ptr.size() - 1;
    const uint64_t nnz = c.idx.size();
    if (n_cols == 0) return OG_OK;
    DevBuf dptr, didx, dval, dm, db, stage;
    OG_ALLOC(ctx, dptr, 4ull * (n_cols + 1)); OG_ALLOC(ctx, didx, 4 * nnz); OG_ALLOC(ctx, dval, 32 * nnz);
    OG_ALLOC(ctx, dm, PB * n_cols); OG_ALLOC(ctx, db, PB * n_cols);
    OG_CUDA(ctx, cudaMemcpyAsync(dptr.p, c.ptr.data(), 4ull * (n_cols + 1), cudaMemcpyHostToDevice, ctx->stream));
    if (nnz) {
        OG_CUDA(ctx, cudaMemcpyAsync(didx.p, c.idx.data(), 4 * nnz, cudaMemcpyHostToDevice, ctx->stream));
        OG_CUDA(ctx, cudaMemcpyAsync(dval.p, c.val.data(), 32 * nnz, cudaMemcpyHostToDevice, ctx->stream));
    }
    OG_LAUNCH(ctx, k_colsum<F>, blocks(n_cols, 128), 128, 0, d_pts, dptr.as<uint32_t>(), didx.as<uint32_t>(), dval.as<uint32_t>(), n_cols,
              COL_HEAVY, dm.as<Affine<F>>());
    OG_TRY(points_mont_to_bytes(ctx, dm.as<Affine<F>>(), n_cols, db.as<uint8_t>()));
    uint32_t longest = 0;
    for (uint32_t i = 0; i < n_cols; i++) longest = std::max(longest, c.ptr[i + 1] - c.ptr[i]);
    if (longest > COL_HEAVY) {
        OG_ALLOC(ctx, stage, PB * longest);
        for (uint32_t i = 0; i < n_cols; i++) {
            const uint32_t b = c.ptr[i], n = c.ptr[i + 1] - b;
            if (n <= COL_HEAVY) continue;
            OG_LAUNCH(ctx, k_gather_rows, blocks(n, 128), 128, 0, d_pts_bytes, (uint32_t)PB, didx.as<uint32_t>() + b, n, stage.as<uint8_t>());
            OG_TRY(msm_dev<F>(ctx, stage.as<uint8_t>(), dval.as<uint8_t>() + 32ull * b, n, db.as<uint8_t>() + PB * i));
        }
    }
    OG_CUDA(ctx, cudaMemcpyAsync(out_host, db.p, PB * n_cols, cudaMemcpyDeviceToHost, ctx->stream));
    OG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return OG_OK;
}

int32_t ptau_prepare(og_ctx* ctx, const uint8_t* acc, uint64_t acc_len, const R1cs& cs, uint32_t depth, uint8_t* pk_out, uint64_t* pk_len,
                     uint8_t* vk_out, uint64_t* vk_len) {
    PtLayout L;
    if (!pk_len || !vk_len || !pt_layout(acc, acc_len, L)) return OG_E_INVALID;
    const uint32_t nv = cs.n_vars, n_pub = cs.n_pub, nc = cs.n_constraints();
    const uint32_t log_m = groth16_domain_log(nc, n_pub);
    const uint64_t m = 1ull << log_m;
    if (log_m > L.log_max) return OG_E_INVALID;
    uint64_t need_pk, need_vk;
    key_sizes(cs, &need_pk, &need_vk);
    if (!pk_out || !vk_out) { *pk_len = need_pk; *vk_len = need_vk; return OG_OK; }
    if (*pk_len < need_pk || *vk_len < need_vk) return OG_E_INVALID;

    // Lagrange bases: P1 = [L_j]_1 | [alpha L_j]_1 | [beta L_j]_1 (m each), H2 = the size-2m basis, Q2 = [L_j]_2
    DevBuf db, P1, P1b, H2, Q2, Q2b;
    OG_ALLOC(ctx, db, acc_len);
    OG_ALLOC(ctx, P1, sizeof(G1Affine) * 3 * m); OG_ALLOC(ctx, P1b, 64 * 3 * m); OG_ALLOC(ctx, H2, sizeof(G1Affine) * 2 * m);
    OG_ALLOC(ctx, Q2, sizeof(G2Affine) * m); OG_ALLOC(ctx, Q2b, 128 * m);
    OG_TRY(clear_flag(ctx));
    OG_CUDA(ctx, cudaMemcpyAsync(db.p, acc, acc_len, cudaMemcpyHostToDevice, ctx->stream));
    const uint8_t* d = db.as<uint8_t>();
    G1Affine* p1 = P1.as<G1Affine>();
    OG_TRY(points_bytes_to_mont(ctx, d + L.tau1, m, p1));
    OG_TRY(points_bytes_to_mont(ctx, d + L.alpha1, m, p1 + m));
    OG_TRY(points_bytes_to_mont(ctx, d + L.beta1, m, p1 + 2 * m));
    OG_TRY(points_bytes_to_mont(ctx, d + L.tau1, 2 * m, H2.as<G1Affine>()));
    OG_TRY(points_bytes_to_mont(ctx, d + L.tau2, m, Q2.as<G2Affine>()));
    OG_TRY(check_flag(ctx));
    for (int k = 0; k < 3; k++) OG_TRY(intt<Fq>(ctx, p1 + k * m, log_m));
    OG_TRY(intt<Fq>(ctx, H2.as<G1Affine>(), log_m + 1));
    OG_TRY(intt<Fq2>(ctx, Q2.as<G2Affine>(), log_m));
    OG_TRY(points_mont_to_bytes(ctx, p1, 3 * m, P1b.as<uint8_t>()));
    OG_TRY(points_mont_to_bytes(ctx, Q2.as<G2Affine>(), m, Q2b.as<uint8_t>()));
    OG_TRY(points_mont_to_bytes(ctx, H2.as<G1Affine>(), 2 * m, db.as<uint8_t>()));   // the accumulator copy is no longer needed
    std::vector<uint8_t> h2(64 * 2 * m), qh(64 * m);
    OG_CUDA(ctx, cudaMemcpyAsync(h2.data(), db.p, 64 * 2 * m, cudaMemcpyDeviceToHost, ctx->stream));
    OG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    for (uint64_t j = 0; j < m; j++) memcpy(&qh[64 * j], &h2[64 * (2 * j + 1)], 64);   // H_query[j] = L^(2m)_(2j+1)

    // column sums over the R1CS (A with its input-consistency rows nc + i, i <= n_pub)
    Csr A = cs.A;
    for (uint32_t i = 0; i <= n_pub; i++) { A.col.push_back(i); A.val.push_back(Fr::one()); A.row_ptr.push_back((uint32_t)A.col.size()); }
    std::vector<Term> ta, tb, tl;
    csr_terms(A, 0, ta);
    csr_terms(cs.B, 0, tb);
    csr_terms(A, (uint32_t)(2 * m), tl); csr_terms(cs.B, (uint32_t)m, tl); csr_terms(cs.C, 0, tl);
    const Cols ca = transpose(nv, ta), cb = transpose(nv, tb), cl = transpose(nv, tl);
    std::vector<uint8_t> qa(64ull * nv), qb1(64ull * nv), qb2(128ull * nv), qlic(64ull * nv);
    OG_TRY(column_sums<Fq>(ctx, p1, P1b.as<uint8_t>(), ca, qa.data()));
    OG_TRY(column_sums<Fq>(ctx, p1, P1b.as<uint8_t>(), cb, qb1.data()));
    OG_TRY(column_sums<Fq2>(ctx, Q2.as<G2Affine>(), Q2b.as<uint8_t>(), cb, qb2.data()));
    OG_TRY(column_sums<Fq>(ctx, p1, P1b.as<uint8_t>(), cl, qlic.data()));

    KeyPoints P;
    P.alpha1 = acc + L.alpha1; P.beta1 = acc + L.beta1; P.delta1 = acc + L.tau1;           // delta = 1: the generators
    P.qa = qa.data(); P.qb1 = qb1.data(); P.ic = qlic.data(); P.ql = qlic.data() + 64ull * (n_pub + 1); P.qh = qh.data();
    P.beta2 = acc + L.beta2; P.delta2 = acc + L.tau2; P.gamma2 = acc + L.tau2; P.qb2 = qb2.data();
    return write_keys(cs, depth, P, pk_out, pk_len, vk_out, vk_len);
}

// ---- phase 2 --------------------------------------------------------------------------------------------------------
static void key_hash(const uint8_t* pk, uint64_t pk_len, const uint8_t* vk, uint64_t vk_len, uint8_t h[32]) {
    std::vector<uint8_t> m(pk, pk + pk_len);
    m.insert(m.end(), vk, vk + vk_len);
    keccak256(m.data(), m.size(), h);
}

static bool vk_matches(const PkLayout& L, const uint8_t* vk, uint64_t vk_len) {
    return vk && vk_len == 12 + 64 + 3 * 128 + 64ull * (L.n_pub + 1) && memcmp(vk, "OGVK", 4) == 0;
}

int32_t phase2_contribute(og_ctx* ctx, const uint8_t* pk, uint64_t pk_len, const uint8_t* vk, uint64_t vk_len, const uint8_t* d32,
                          const uint8_t* nonce32, uint8_t* pk_out, uint64_t* pk_out_len, uint8_t* vk_out, uint64_t* vk_out_len,
                          uint8_t* rec_out, uint64_t* rec_len) {
    PkLayout L;
    if (!pk_out_len || !vk_out_len || !rec_len || !pk || !pk_layout(pk, pk_len, L) || !vk_matches(L, vk, vk_len)) return OG_E_INVALID;
    if (!pk_out || !vk_out || !rec_out) { *pk_out_len = pk_len; *vk_out_len = vk_len; *rec_len = DR_BYTES; return OG_OK; }
    if (*pk_out_len < pk_len || *vk_out_len < vk_len || *rec_len < DR_BYTES || !d32 || !nonce32) return OG_E_INVALID;
    Fr dd, k, dinv;
    int32_t rc = OG_OK;
    if (!host_load(dd, d32) || !host_load(k, nonce32)) rc = OG_E_ENCODING;
    else if (dd.is_zero() || k.is_zero()) rc = OG_E_INVALID;
    if (rc == OG_OK) {
        rc = [&]() -> int32_t {
            dinv = dd.inv();
            memcpy(pk_out, pk, pk_len);
            memcpy(vk_out, vk, vk_len);
            const uint64_t n_lh = (L.qh - L.ql) / 64 + (1ull << L.log_m);          // L and H are adjacent
            OG_TRY(scale_bytes_host<Fq>(ctx, pk + L.ql, n_lh, dinv, pk_out + L.ql));
            OG_TRY(scale_bytes_host<Fq>(ctx, pk + L.delta1, 1, dd, pk_out + L.delta1));
            OG_TRY(scale_bytes_host<Fq2>(ctx, pk + L.delta2, 1, dd, pk_out + L.delta2));
            memcpy(vk_out + VK_DELTA2, pk_out + L.delta2, 128);
            memcpy(rec_out, "OGDR", 4);
            const uint32_t ver = 1;
            memcpy(rec_out + 4, &ver, 4);
            key_hash(pk, pk_len, vk, vk_len, rec_out + 8);
            return make_poks(ctx, rec_out + 8, &dd, &k, 1, rec_out + 40);
        }();
    }
    wipe(&dd, sizeof(dd)); wipe(&k, sizeof(k)); wipe(&dinv, sizeof(dinv));
    if (rc == OG_OK) { *pk_out_len = pk_len; *vk_out_len = vk_len; *rec_len = DR_BYTES; }
    return rc;
}

int32_t phase2_verify(og_ctx* ctx, const uint8_t* pk0, uint64_t pk0_len, const uint8_t* vk0, uint64_t vk0_len, const uint8_t* pk1,
                      uint64_t pk1_len, const uint8_t* vk1, uint64_t vk1_len, const uint8_t* rec, uint64_t rec_len) {
    PkLayout L, L1;
    if (!pk0 || !pk1 || !pk_layout(pk0, pk0_len, L) || !pk_layout(pk1, pk1_len, L1) || pk0_len != pk1_len || vk0_len != vk1_len ||
        !vk_matches(L, vk0, vk0_len) || !vk_matches(L, vk1, vk1_len)) return OG_E_VERIFY;
    // every byte outside delta, L and H unchanged; the vk's delta_2 is the pk's
    const uint64_t end_h = L.qh + (64ull << L.log_m);
    if (memcmp(pk0, pk1, L.delta1) != 0 || memcmp(pk0 + L.qa, pk1 + L.qa, L.ql - L.qa) != 0 ||
        memcmp(pk0 + end_h, pk1 + end_h, pk0_len - end_h) != 0 || memcmp(vk0, vk1, VK_DELTA2) != 0 ||
        memcmp(vk0 + VK_DELTA2 + 128, vk1 + VK_DELTA2 + 128, vk0_len - VK_DELTA2 - 128) != 0 ||
        memcmp(vk1 + VK_DELTA2, pk1 + L.delta2, 128) != 0 || memcmp(vk0 + VK_DELTA2, pk0 + L.delta2, 128) != 0) return OG_E_VERIFY;
    if (!rec || rec_len != DR_BYTES || memcmp(rec, "OGDR", 4) != 0) return OG_E_VERIFY;
    uint32_t ver;
    memcpy(&ver, rec + 4, 4);
    uint8_t h[32];
    key_hash(pk0, pk0_len, vk0, vk0_len, h);
    if (ver != 1 || memcmp(h, rec + 8, 32) != 0) return OG_E_VERIFY;
    uint8_t g1b[64], g2b[128];
    OG_TRY(generators(ctx, g1b, g2b));
    G1Affine g1; G2Affine g2;
    load_g1(g1, g1b); load_g2(g2, g2b);
    G1Affine D1; G2Affine D2;
    if (!check_pok(rec + 8, 0, rec + 40, g1, g2, D1, D2)) return OG_E_VERIFY;
    G1Affine od1, nd1; G2Affine od2, nd2;
    if (!load_g1(od1, pk0 + L.delta1) || !load_g1(nd1, pk1 + L.delta1) || !load_g2(od2, pk0 + L.delta2) || !load_g2(nd2, pk1 + L.delta2) ||
        nd1.is_inf() || nd2.is_inf()) return OG_E_VERIFY;
    if (!pair_eq(nd1, g2, od1, D2) || !pair_eq(nd1, g2, g1, nd2)) return OG_E_VERIFY;
    // L || H: e(sum rho^i new_i, new delta_2) == e(sum rho^i old_i, old delta_2)
    const uint64_t n_lh = (end_h - L.ql) / 64;
    DevBuf db, out, rho;
    OG_ALLOC(ctx, db, 2 * 64 * n_lh); OG_ALLOC(ctx, out, 128);
    OG_CUDA(ctx, cudaMemcpyAsync(db.p, pk0 + L.ql, 64 * n_lh, cudaMemcpyHostToDevice, ctx->stream));
    OG_CUDA(ctx, cudaMemcpyAsync(db.as<uint8_t>() + 64 * n_lh, pk1 + L.ql, 64 * n_lh, cudaMemcpyHostToDevice, ctx->stream));
    bool ok;
    OG_TRY(check_points<Fq>(ctx, db.as<uint8_t>() + 64 * n_lh, n_lh, 1, &ok));
    if (!ok) return OG_E_VERIFY;
    std::vector<uint8_t> k1(pk1, pk1 + pk1_len);
    k1.insert(k1.end(), vk1, vk1 + vk1_len);
    std::vector<uint8_t> k0(pk0, pk0 + pk0_len);
    k0.insert(k0.end(), vk0, vk0 + vk0_len);
    OG_TRY(rho_powers(ctx, fs_rho(k0.data(), k0.size(), k1.data(), k1.size(), rec, rec_len), n_lh, rho));
    OG_TRY(msm_dev<Fq>(ctx, db.as<uint8_t>(), rho.as<uint8_t>(), n_lh, out.as<uint8_t>()));
    OG_TRY(msm_dev<Fq>(ctx, db.as<uint8_t>() + 64 * n_lh, rho.as<uint8_t>(), n_lh, out.as<uint8_t>() + 64));
    uint8_t s[128];
    OG_CUDA(ctx, cudaMemcpyAsync(s, out.p, 128, cudaMemcpyDeviceToHost, ctx->stream));
    OG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    G1Affine S0, S1;
    if (!load_g1(S0, s) || !load_g1(S1, s + 64) || !pair_eq(S1, nd2, S0, od2)) return OG_E_VERIFY;
    return OG_OK;
}

// ---- kernel-level entry points --------------------------------------------------------------------------------------
int32_t scale_points_dev(og_ctx* ctx, int g2, const uint8_t* d_points, const uint8_t* d_scalars, uint64_t n, int per_point, uint8_t* d_out) {
    if (n == 0) return OG_OK;
    const uint64_t ns = per_point ? n : 1;
    DevBuf s, pm;
    OG_ALLOC(ctx, s, sizeof(Fr) * ns);
    OG_ALLOC(ctx, pm, (g2 ? sizeof(G2Affine) : sizeof(G1Affine)) * n);
    OG_TRY(mimc_to_mont_dev(ctx, d_scalars, ns, s.as<Fr>()));
    if (g2) {
        OG_TRY(points_bytes_to_mont(ctx, d_points, n, pm.as<G2Affine>()));
        OG_TRY(scale<Fq2>(ctx, pm.as<G2Affine>(), s.as<Fr>(), n, per_point, pm.as<G2Affine>()));
        OG_TRY(points_mont_to_bytes(ctx, pm.as<G2Affine>(), n, d_out));
    } else {
        OG_TRY(points_bytes_to_mont(ctx, d_points, n, pm.as<G1Affine>()));
        OG_TRY(scale<Fq>(ctx, pm.as<G1Affine>(), s.as<Fr>(), n, per_point, pm.as<G1Affine>()));
        OG_TRY(points_mont_to_bytes(ctx, pm.as<G1Affine>(), n, d_out));
    }
    OG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return OG_OK;
}

int32_t intt_points_dev(og_ctx* ctx, int g2, uint8_t* d_points, uint32_t log_m) {
    const uint64_t m = 1ull << log_m;
    DevBuf pm;
    OG_ALLOC(ctx, pm, (g2 ? sizeof(G2Affine) : sizeof(G1Affine)) * m);
    if (g2) {
        OG_TRY(points_bytes_to_mont(ctx, d_points, m, pm.as<G2Affine>()));
        OG_TRY(intt<Fq2>(ctx, pm.as<G2Affine>(), log_m));
        OG_TRY(points_mont_to_bytes(ctx, pm.as<G2Affine>(), m, d_points));
    } else {
        OG_TRY(points_bytes_to_mont(ctx, d_points, m, pm.as<G1Affine>()));
        OG_TRY(intt<Fq>(ctx, pm.as<G1Affine>(), log_m));
        OG_TRY(points_mont_to_bytes(ctx, pm.as<G1Affine>(), m, d_points));
    }
    OG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return OG_OK;
}

}  // namespace og
