// owshen_b200/csrc/mimc.cu -- MiMC7 (circomlib flavour) on sm_90a: 2-to-1 node hash, batched Merkle
// paths (BASELINE config 2), level-by-level tree build, the note hashes (k_note_hash), and the witness generators
// of the withdraw, deposit, transfer, association, exclusion, labeled and labeled association withdraw and owned transfer
// statements (every t^2, t^4, t^6, t^7 of every round is a circuit variable).
//
// Not in the reference (its only field "hash" is a placeholder product,
// /root/reference/src/blockchain/tx/owshen_airdrop/babyjubjub/mod.rs:202-204); the algorithm is the
// published circomlib one, see DESIGN.md section 2.  One thread owns one sequential hash chain:
// a path is 32 levels x 2 permutations x 91 rounds x 4 multiplications that each depend on the
// previous one, so the parallelism is across paths, the arithmetic stays in registers and the
// kernel is bound by the integer multiply-add pipe, not by HBM (DESIGN.md section 5.2).
#include "common.cuh"
#include "host_math.hpp"
#include "mimc.cuh"
#include "mimc_core.cuh"
#include <iterator>
#include <stdlib.h>
#include <utility>

namespace og {

__constant__ uint32_t c_mimc[MIMC_ROUNDS * 8];   // round constants, Montgomery form

__device__ __forceinline__ Fr mimc_c(int i) {
    Fr r;
#pragma unroll
    for (int j = 0; j < 8; j++) r.l[j] = c_mimc[i * 8 + j];
    return r;
}

// hash(x, k) = perm(x, k) + k.  TRACE: also store t2,t4,t6,t7 of every round to trace[4*i..].
template <bool TRACE>
__device__ __forceinline__ Fr mimc7_hash(const Fr& x, const Fr& k, Fr* trace) {
    Fr r = x;
#pragma unroll 1
    for (int i = 0; i < MIMC_ROUNDS; i++) {
        Fr t = r + k + mimc_c(i);
        Fr t2 = t.sqr();
        if (TRACE) {
            Fr t4 = t2.sqr();
            Fr t6 = t4 * t2;
            r = t6 * t;
            trace[4 * i] = t2; trace[4 * i + 1] = t4; trace[4 * i + 2] = t6; trace[4 * i + 3] = r;
        } else {
            // same value, shallower dependency chain: t3 and t4 are independent
            Fr t3 = t2 * t;
            Fr t4 = t2.sqr();
            r = t3 * t4;
        }
    }
    return r + k;
}

// MultiMiMC7([l, r], key 0): r1 = l + hash(l, 0); out = r1 + r + hash(r, r1).  The TRACE form (witness generation) stores
// every fully reduced intermediate; the plain form is the lazy chain of mimc_core.cuh.
template <bool TRACE>
__device__ __forceinline__ Fr mimc7_hash2(const Fr& l, const Fr& r, Fr* trace1, Fr* trace2) {
    if (!TRACE) return mimc7_hash2_lazy(l, r, [](int i) { return mimc_c(i); });
    Fr r1 = l + mimc7_hash<TRACE>(l, Fr::zero(), trace1);
    return r1 + r + mimc7_hash<TRACE>(r, r1, trace2);
}

__global__ void __launch_bounds__(64) k_hash2(const uint8_t* __restrict__ left, const uint8_t* __restrict__ right,
                                              uint64_t n, uint8_t* __restrict__ out, int* flag) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Fr l = load_canonical<Fr>(left + 32 * i, flag);
    Fr r = load_canonical<Fr>(right + 32 * i, flag);
    store_canonical(out + 32 * i, mimc7_hash2<false>(l, r, nullptr, nullptr));
}

// one level of a full tree: out[i] = hash2(in[2i], in[2i+1]), Montgomery-form in and out
__global__ void __launch_bounds__(64) k_tree_level(const Fr* __restrict__ in, uint64_t n_out, Fr* __restrict__ out) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_out) return;
    out[i] = mimc7_hash2<false>(in[2 * i], in[2 * i + 1], nullptr, nullptr);
}

// one level of an APPEND to a fixed-depth sparse tree: parents [p0, p0 + n_out) of the dirty children [c0, c0 + n_in).
// A child left of the dirty range is the stored boundary node of this level (at most one: index c0 - 1), a child right
// of it is the empty-subtree root of the level (append-only: nothing exists to the right of the new leaves).
__global__ void __launch_bounds__(64) k_tree_append_level(const Fr* __restrict__ in, uint64_t c0, uint64_t n_in, uint64_t p0, uint64_t n_out,
                                                          Fr left_boundary, Fr zero, Fr* __restrict__ out) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_out) return;
    uint64_t l = 2 * (p0 + i), r = l + 1;
    Fr a = l < c0 ? left_boundary : (l < c0 + n_in ? in[l - c0] : zero);
    Fr b = r < c0 ? left_boundary : (r < c0 + n_in ? in[r - c0] : zero);
    out[i] = mimc7_hash2<false>(a, b, nullptr, nullptr);
}

__global__ void __launch_bounds__(128) k_to_mont(const uint8_t* __restrict__ in, uint64_t n, Fr* __restrict__ out, int* flag) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = load_canonical<Fr>(in + 32 * i, flag);
}
__global__ void __launch_bounds__(128) k_from_mont(const Fr* __restrict__ in, uint64_t n, uint8_t* __restrict__ out) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) store_canonical(out + 32 * i, in[i]);
}

// BASELINE config 2.  One thread per path; 32 threads per CTA so that 4096 paths spread over
// 128 SMs instead of piling 4 warps onto 32 of them (the chain is latency-bound per warp).
__global__ void __launch_bounds__(32) k_merkle_paths(const uint8_t* __restrict__ leaves, const uint8_t* __restrict__ siblings,
                                                     const uint32_t* __restrict__ path_bits, uint32_t n_paths, uint32_t depth,
                                                     uint8_t* __restrict__ out_nodes, int* flag) {
    uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n_paths) return;
    Fr cur = load_canonical<Fr>(leaves + 32ull * p, flag);
    uint8_t* o = out_nodes + (uint64_t)p * (depth + 1) * 32;
    store_canonical(o, cur);
    uint32_t bits = path_bits[p];
    const uint8_t* sp = siblings + (uint64_t)p * depth * 32;
#pragma unroll 1
    for (uint32_t l = 0; l < depth; l++) {
        Fr sib = load_canonical<Fr>(sp + 32 * l, flag);
        bool right = (bits >> l) & 1;
        Fr a = right ? sib : cur;
        Fr b = right ? cur : sib;
        cur = mimc7_hash2<false>(a, b, nullptr, nullptr);
        store_canonical(o + 32 * (l + 1), cur);
    }
}

// The witness of a Merkle path from the leaf `cur`: `depth` level blocks (sibling, bit, left, perm1[perm], perm2[perm], out)
// written from v on, lvl_size elements apart, with the siblings from sp (32 B canonical each) and bit l of `bits` set when
// the node is a right child.  Returns the root.  Shared by the withdraw, transfer, association and exclusion witness kernels.
__device__ __forceinline__ Fr witness_path(Fr cur, Fr* v, uint32_t depth, uint32_t lvl_size, uint32_t perm, const uint8_t* sp,
                                           uint32_t bits, int* flag) {
    const Fr one = Fr::one();
#pragma unroll 1
    for (uint32_t l = 0; l < depth; l++) {
        Fr* lv = v + l * lvl_size;
        Fr sib = load_canonical<Fr>(sp + 32 * l, flag);
        bool right = (bits >> l) & 1;
        Fr a = right ? sib : cur;
        Fr b = right ? cur : sib;
        lv[0] = sib;
        lv[1] = right ? one : Fr::zero();
        lv[2] = a;
        cur = mimc7_hash2<true>(a, b, lv + 3, lv + 3 + perm);
        lv[3 + 2 * perm] = cur;
    }
    return cur;
}

// Witness of the withdraw statement, layout of DESIGN.md section 3 (== oracle/withdraw_circuit.py).
// One thread per proof; W is [batch][n_vars] in Montgomery form.
__global__ void __launch_bounds__(32) k_withdraw_witness(WithdrawLayout L, uint32_t w_stride, const uint8_t* __restrict__ nullifiers,
                                                         const uint8_t* __restrict__ secrets, const uint8_t* __restrict__ recipients,
                                                         const uint8_t* __restrict__ siblings, const uint32_t* __restrict__ path_bits,
                                                         uint32_t batch, Fr* __restrict__ W, int* flag) {
    uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= batch) return;
    Fr* w = W + (uint64_t)p * w_stride;
    Fr nu = load_canonical<Fr>(nullifiers + 32ull * p, flag);
    Fr se = load_canonical<Fr>(secrets + 32ull * p, flag);
    Fr re = load_canonical<Fr>(recipients + 32ull * p, flag);
    Fr one = Fr::one();
    w[0] = one; w[3] = re; w[4] = nu; w[5] = se;
    w[6] = re.sqr();
    // nullifier_hash = MultiMiMC7([nullifier], key 1) = 1 + nullifier + hash(nullifier, 1)
    w[2] = one + nu + mimc7_hash<true>(nu, one, w + 7);
    Fr cur = mimc7_hash2<true>(nu, se, w + L.cm_base, w + L.cm_base + L.perm);
    w[L.cm_out] = cur;
    w[1] = witness_path(cur, w + L.lvl_base, L.depth, L.lvl_size, L.perm, siblings + (uint64_t)p * L.depth * 32, path_bits[p], flag);
}

// Witness of the deposit statement, layout of DESIGN.md section 3 (== oracle/deposit_circuit.py).
// One thread per proof; row p starts at W + p * w_stride, Montgomery form.
__global__ void __launch_bounds__(32) k_deposit_witness(DepositLayout L, uint32_t w_stride, const uint8_t* __restrict__ nullifiers,
                                                        const uint8_t* __restrict__ secrets, const uint8_t* __restrict__ depositors,
                                                        uint32_t batch, Fr* __restrict__ W, int* flag) {
    uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= batch) return;
    Fr* w = W + (uint64_t)p * w_stride;
    Fr nu = load_canonical<Fr>(nullifiers + 32ull * p, flag);
    Fr se = load_canonical<Fr>(secrets + 32ull * p, flag);
    Fr de = load_canonical<Fr>(depositors + 32ull * p, flag);
    w[0] = Fr::one(); w[2] = de; w[3] = nu; w[4] = se;
    w[5] = de.sqr();
    Fr cm = mimc7_hash2<true>(nu, se, w + L.cm_base, w + L.cm_base + L.perm);
    w[L.cm_out] = cm;
    w[1] = cm;
}

// A note's amount (< 2^64), its 64 bits and its commitment MultiMiMC7([nullifier, secret, token, amount], 0), every round
// value written into the note block v.  Returns the commitment.
__device__ __forceinline__ Fr transfer_note(const TransferLayout& L, Fr* v, const Fr& nu, const Fr& se, const Fr& token, uint64_t amount,
                                            uint32_t cm, uint32_t cm_out) {
    const Fr one = Fr::one(), zero = Fr::zero();
    uint32_t c[8] = {(uint32_t)amount, (uint32_t)(amount >> 32), 0, 0, 0, 0, 0, 0};
    Fr am = Fr::from_canonical(c);
    v[0] = nu; v[1] = se; v[2] = am;
#pragma unroll 8
    for (uint32_t k = 0; k < TRANSFER_AMOUNT_BITS; k++) v[3 + k] = ((amount >> k) & 1) ? one : zero;
    const Fr xs[4] = {nu, se, token, am};
    Fr r = zero;
#pragma unroll 1
    for (int k = 0; k < 4; k++) r = r + xs[k] + mimc7_hash<true>(xs[k], r, v + cm + k * L.perm);
    v[cm_out] = r;
    return r;
}

// Witness of the transfer statement, layout of DESIGN.md section 3 (== oracle/transfer_circuit.py); row p starts at
// W + p * w_stride, Montgomery form.  A CTA covers 32 proofs with four warps, one per independent hash chain of a proof, so
// no warp diverges and a proof's critical path is one input's commitment and Merkle path (4 + 2 * depth permutations, about
// one withdraw path):
//   warps 0, 1   input i: amount bits, commitment, the depth levels
//   warps 2, 3   input j - 2's nullifier hash, then output j - 2: amount bits, commitment
// After the barrier, warp 0 writes the proof's remaining scalars (public amount, recipient, nh_diff_inv).
__global__ void __launch_bounds__(128) k_transfer_witness(TransferLayout L, uint32_t w_stride, TransferInputs in, uint32_t batch,
                                                          Fr* __restrict__ W, int* flag) {
    const uint32_t role = threadIdx.x >> 5;
    const uint32_t p = blockIdx.x * 32 + (threadIdx.x & 31);
    const bool active = p < batch;
    Fr* w = W + (uint64_t)p * w_stride;
    const Fr one = Fr::one();
    if (active) {
        const Fr token = load_canonical<Fr>(in.tokens + 32ull * p, flag);
        if (role < 2) {
            const uint32_t i = role;
            Fr* v = w + L.inp(i);
            Fr nu = load_canonical<Fr>(in.in_null + 64ull * p + 32 * i, flag);
            Fr se = load_canonical<Fr>(in.in_sec + 64ull * p + 32 * i, flag);
            Fr cur = transfer_note(L, v, nu, se, token, in.in_amounts[2ull * p + i], L.in_cm, L.in_cm_out);
            witness_path(cur, v + L.lvl_base, L.depth, L.lvl_size, L.perm, in.in_sib + 32ull * L.depth * (2ull * p + i),
                         in.in_bits[2ull * p + i], flag);
        } else {
            const uint32_t j = role - 2;
            // nullifier_hash = MultiMiMC7([nullifier], key 1) = 1 + nullifier + hash(nullifier, 1), as in withdraw
            Fr* v = w + L.inp(j);
            Fr nu = load_canonical<Fr>(in.in_null + 64ull * p + 32 * j, flag);
            w[5 + j] = one + nu + mimc7_hash<true>(nu, one, v + L.nh_perm);
            Fr* o = w + L.out(j);
            Fr onu = load_canonical<Fr>(in.out_null + 64ull * p + 32 * j, flag);
            Fr ose = load_canonical<Fr>(in.out_sec + 64ull * p + 32 * j, flag);
            w[7 + j] = transfer_note(L, o, onu, ose, token, in.out_amounts[2ull * p + j], L.out_cm, L.out_cm_out);
        }
        if (role == 0) {
            Fr re = load_canonical<Fr>(in.recipients + 32ull * p, flag);
            w[0] = one;
            w[1] = load_canonical<Fr>(in.roots + 32ull * p, flag);
            w[3] = token; w[4] = re;
            w[9] = re.sqr();
        }
    }
    __syncthreads();   // warps 1..3 wrote the amounts and nullifier hashes read below
    if (active && role == 0) {
        Fr a_in = w[L.inp(0) + 2] + w[L.inp(1) + 2], a_out = w[L.out(0) + 2] + w[L.out(1) + 2];
        w[2] = a_out - a_in;
        w[10] = (w[5] - w[6]).inv();   // inv(0) = 0: two inputs with one nullifier leave the row unsatisfiable
    }
}

// The withdraw chain of the association and exclusion statements, whose rows share its variables: ONE, recipient (3),
// nullifier (5), secret (6), recipient_sq (7), the nullifier hash (2) with its permutation just below the commitment block,
// the commitment with its round values, the pool path from L.pool_base, root (1).
template <class Layout>
__device__ __forceinline__ void withdraw_chain_witness(const Layout& L, Fr* w, const Fr& nu, const Fr& se, const uint8_t* recipient,
                                                       const uint8_t* sp, uint32_t bits, int* flag) {
    Fr re = load_canonical<Fr>(recipient, flag);
    Fr one = Fr::one();
    w[0] = one; w[3] = re; w[5] = nu; w[6] = se;
    w[7] = re.sqr();
    // nullifier_hash = MultiMiMC7([nullifier], key 1) = 1 + nullifier + hash(nullifier, 1), as in withdraw
    w[2] = one + nu + mimc7_hash<true>(nu, one, w + L.cm_base - L.perm);
    Fr cm = mimc7_hash2<true>(nu, se, w + L.cm_base, w + L.cm_base + L.perm);
    w[L.cm_out] = cm;
    w[1] = witness_path(cm, w + L.pool_base, L.depth, L.lvl_size, L.perm, sp, bits, flag);
}

// Witness of the association-set withdraw statement, layout of DESIGN.md section 3 (== oracle/association_circuit.py); row p
// starts at W + p * w_stride, Montgomery form.  A CTA covers 32 proofs with two warps, one per independent chain of a proof,
// so no warp diverges and a proof's critical path stays at about one withdraw path:
//   warp 0   ONE, recipient, recipient_sq, the nullifier hash, the commitment with its round values, the pool path, root
//   warp 1   the commitment again in registers (no stores), the association path, association_root
// The warps write disjoint variables, so no barrier is needed.
__global__ void __launch_bounds__(64) k_association_witness(AssociationLayout L, uint32_t w_stride, AssociationInputs in, uint32_t batch,
                                                            Fr* __restrict__ W, int* flag) {
    const uint32_t role = threadIdx.x >> 5;
    const uint32_t p = blockIdx.x * 32 + (threadIdx.x & 31);
    if (p >= batch) return;
    Fr* w = W + (uint64_t)p * w_stride;
    Fr nu = load_canonical<Fr>(in.nullifiers + 32ull * p, flag);
    Fr se = load_canonical<Fr>(in.secrets + 32ull * p, flag);
    if (role == 0) {
        withdraw_chain_witness(L, w, nu, se, in.recipients + 32ull * p, in.siblings + 32ull * L.depth * p, in.path_bits[p], flag);
    } else {
        Fr cm = mimc7_hash2<false>(nu, se, nullptr, nullptr);
        w[4] = witness_path(cm, w + L.assoc_base, L.depth, L.lvl_size, L.perm, in.assoc_siblings + 32ull * L.depth * p,
                            in.assoc_path_bits[p], flag);
    }
}

constexpr uint64_t R_LO64 = 0x43e1f593f0000001ull;   // r mod 2^64

// the 33 low bits of the canonical representative of (a - b - 1) mod r, for a, b < 2^64: when a <= b the difference is
// r - (b + 1 - a), whose low 64 bits are r's low 64 bits minus (b + 1 - a), all mod 2^64
__device__ __forceinline__ uint64_t gap_bits(uint64_t a, uint64_t b) {
    return a - b - 1 + (a > b ? 0 : R_LO64);
}

// likewise the 64 low bits of the canonical (a - b) mod r
__device__ __forceinline__ uint64_t diff_bits(uint64_t a, uint64_t b) {
    return a - b + (a >= b ? 0 : R_LO64);
}

// the n_bits low bits of v as field elements 0 / 1, LSB first
__device__ __forceinline__ void store_range_bits(Fr* out, uint64_t v, uint32_t n_bits = EXCLUSION_RANGE_BITS) {
    const Fr one = Fr::one(), zero = Fr::zero();
#pragma unroll 1
    for (uint32_t k = 0; k < n_bits; k++) out[k] = ((v >> k) & 1) ? one : zero;
}

// Witness of the exclusion withdraw statement, layout of DESIGN.md section 3 (== oracle/exclusion_circuit.py); row p starts
// at W + p * w_stride, Montgomery form.  A CTA covers 32 proofs with two warps, one per independent chain of a proof, so no
// warp diverges and a proof's critical path stays at about one withdraw path:
//   warp 0   the withdraw chain (withdraw_chain_witness): 67 permutations at depth 32
//   warp 1   low and next, the low / next / gap_lo / gap_hi bits from integer arithmetic on the path word, the blocklist
//            leaf MultiMiMC7([low, next], 0) with its round values, the exclusion path, exclusion_root: 66 permutations
// The warps write disjoint variables, so no barrier is needed.  Only the low `depth` bits of the path word count, as in
// witness_path; x = 1 + that index is at most 2^32.
__global__ void __launch_bounds__(64) k_exclusion_witness(ExclusionLayout L, uint32_t w_stride, ExclusionInputs in, uint32_t batch,
                                                          Fr* __restrict__ W, int* flag) {
    const uint32_t role = threadIdx.x >> 5;
    const uint32_t p = blockIdx.x * 32 + (threadIdx.x & 31);
    if (p >= batch) return;
    Fr* w = W + (uint64_t)p * w_stride;
    if (role == 0) {
        Fr nu = load_canonical<Fr>(in.nullifiers + 32ull * p, flag);
        Fr se = load_canonical<Fr>(in.secrets + 32ull * p, flag);
        withdraw_chain_witness(L, w, nu, se, in.recipients + 32ull * p, in.siblings + 32ull * L.depth * p, in.path_bits[p], flag);
    } else {
        const uint64_t lo = in.low[p], nx = in.next[p];
        const uint64_t mask = L.depth >= 32 ? 0xffffffffull : (1ull << L.depth) - 1;
        const uint64_t x = 1 + (in.path_bits[p] & mask);
        store_range_bits(w + L.low_bits, lo);
        store_range_bits(w + L.next_bits, nx);
        store_range_bits(w + L.gap_lo_bits, gap_bits(x, lo));
        store_range_bits(w + L.gap_hi_bits, gap_bits(nx, x));
        uint32_t c[8] = {(uint32_t)lo, (uint32_t)(lo >> 32), 0, 0, 0, 0, 0, 0};
        const Fr flo = Fr::from_canonical(c);
        c[0] = (uint32_t)nx; c[1] = (uint32_t)(nx >> 32);
        const Fr fnx = Fr::from_canonical(c);
        w[8] = flo; w[9] = fnx;
        Fr leaf = mimc7_hash2<true>(flo, fnx, w + L.leaf_base, w + L.leaf_base + L.perm);
        w[L.leaf_out] = leaf;
        w[4] = witness_path(leaf, w + L.excl_base, L.depth, L.lvl_size, L.perm, in.excl_siblings + 32ull * L.depth * p,
                            in.excl_path_bits[p], flag);
    }
}

__device__ __forceinline__ Fr fr_from_u64(uint64_t v) {
    const uint32_t c[8] = {(uint32_t)v, (uint32_t)(v >> 32), 0, 0, 0, 0, 0, 0};
    return Fr::from_canonical(c);
}

// MultiMiMC7(xs, key): r = key; r = r + x + hash(x, r) per input.  The plain form runs the lazy chain of mimc_core.cuh; the
// TRACE form stores every round value of the k-th permutation from trace + k * perm on.
template <bool TRACE, int N>
__device__ __forceinline__ Fr mimc7_multi_hash(const Fr (&xs)[N], const Fr& key, Fr* trace, uint32_t perm) {
    Fr r = key;
#pragma unroll
    for (int k = 0; k < N; k++) {
        const Fr h = TRACE ? mimc7_hash<true>(xs[k], r, trace + k * perm) : mimc7_perm_lazy<false>(xs[k], r, [](int i) { return mimc_c(i); });
        r = r + xs[k] + h;
    }
    return r;
}

// item i of a note-hash column as a field element
template <NoteColumn COL>
__device__ __forceinline__ Fr note_column(const uint8_t* col, uint64_t i, int* flag) {
    if (COL == COL_FR) return load_canonical<Fr>(col + 32 * i, flag);
    if (COL == COL_U64) return fr_from_u64(reinterpret_cast<const uint64_t*>(col)[i]);
    return Fr::from_u32(reinterpret_cast<const uint32_t*>(col)[i]);
}

template <NoteHash H, size_t... K>
__device__ __forceinline__ Fr note_hash_one(const StatementInputs& cols, uint64_t i, int* flag, std::index_sequence<K...>) {
    const Fr xs[sizeof...(K)] = {note_column<NOTE_HASHES[H].cols[K]>(cols.p[K], i, flag)...};
    return mimc7_multi_hash<false>(xs, Fr::from_u32(NOTE_HASHES[H].key), nullptr, 0);
}

// The note hash H (the note-hash table, mimc.cuh), one thread per item; the row's column count and types are template
// constants, so each instance loads exactly its columns.
template <NoteHash H>
__global__ void __launch_bounds__(64) k_note_hash(StatementInputs cols, uint64_t n, uint8_t* __restrict__ out, int* flag) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    store_canonical(out + 32 * i, note_hash_one<H>(cols, i, flag, std::make_index_sequence<NOTE_HASHES[H].n_cols>{}));
}

// The labeled note's part of the labeled and labeled association witnesses, whose layouts and inputs share the names it
// reads.  labeled_note_witness: nullifier, secret, the precommitment and the leaf with their round values, the pool path,
// root (70 permutations at depth 32).  labeled_change_witness: the public and scalar inputs but variable 4 (the exclusion or
// association root) and variables 15 on, the nullifier hash, the change precommitment and change_commitment with their round
// values (7 permutations), then the amount, withdrawn, change and label bits from integer arithmetic.
template <class Layout, class Inputs>
__device__ __forceinline__ void labeled_note_witness(const Layout& L, Fr* w, const Inputs& in, uint32_t p, int* flag) {
    const Fr key = Fr::from_u32(LABELED_KEY);
    const Fr nu = load_canonical<Fr>(in.nullifiers + 32ull * p, flag);
    const Fr se = load_canonical<Fr>(in.secrets + 32ull * p, flag);
    const Fr token = load_canonical<Fr>(in.tokens + 32ull * p, flag);
    w[8] = nu; w[9] = se;
    const Fr note[2] = {nu, se};
    const Fr pre = mimc7_multi_hash<true>(note, key, w + L.pre_base, L.perm);
    w[L.pre_out] = pre;
    const Fr leaf_in[4] = {pre, token, fr_from_u64(in.amounts[p]), Fr::from_u32(in.labels[p])};
    const Fr leaf = mimc7_multi_hash<true>(leaf_in, key, w + L.leaf_base, L.perm);
    w[L.leaf_out] = leaf;
    w[1] = witness_path(leaf, w + L.pool_base, L.depth, L.lvl_size, L.perm, in.siblings + 32ull * L.depth * p, in.path_bits[p], flag);
}

template <class Layout, class Inputs>
__device__ __forceinline__ void labeled_change_witness(const Layout& L, Fr* w, const Inputs& in, uint32_t p, int* flag) {
    const Fr key = Fr::from_u32(LABELED_KEY);
    const Fr one = Fr::one();
    const Fr token = load_canonical<Fr>(in.tokens + 32ull * p, flag);
    const Fr re = load_canonical<Fr>(in.recipients + 32ull * p, flag);
    const Fr nu = load_canonical<Fr>(in.nullifiers + 32ull * p, flag);
    const Fr cnu = load_canonical<Fr>(in.change_nullifiers + 32ull * p, flag);
    const Fr cse = load_canonical<Fr>(in.change_secrets + 32ull * p, flag);
    const uint64_t amount = in.amounts[p], wd = in.withdrawn[p];
    const uint32_t label = in.labels[p];
    const Fr am = fr_from_u64(amount), fwd = fr_from_u64(wd), la = Fr::from_u32(label), change = am - fwd;
    w[0] = one; w[3] = re; w[5] = token; w[6] = fwd;
    w[10] = re.sqr();
    w[11] = am; w[12] = la; w[13] = cnu; w[14] = cse;
    // nullifier_hash = MultiMiMC7([nullifier], key 1) = 1 + nullifier + hash(nullifier, 1), as in withdraw
    w[2] = one + nu + mimc7_hash<true>(nu, one, w + L.pre_base - L.perm);
    const Fr cnote[2] = {cnu, cse};
    const Fr cpre = mimc7_multi_hash<true>(cnote, key, w + L.cpre_base, L.perm);
    w[L.cpre_out] = cpre;
    const Fr ccm_in[4] = {cpre, token, change, la};
    w[7] = mimc7_multi_hash<true>(ccm_in, key, w + L.ccm_base, L.perm);
    store_range_bits(w + L.amount_bits, amount, LABELED_AMOUNT_BITS);
    store_range_bits(w + L.withdrawn_bits, wd, LABELED_AMOUNT_BITS);
    store_range_bits(w + L.change_bits, diff_bits(amount, wd), LABELED_AMOUNT_BITS);
    store_range_bits(w + L.label_bits, label, LABELED_LABEL_BITS);
}

// Witness of the labeled withdraw statement, layout of DESIGN.md section 3 (== oracle/labeled_circuit.py); row p starts at
// W + p * w_stride, Montgomery form.  A CTA covers 32 proofs with three warps, one per independent chain of a proof, so no
// warp diverges and a proof's critical path stays at about one withdraw path:
//   warp 0   labeled_note_witness: 70 permutations at depth 32
//   warp 1   low and next, the blocklist leaf MultiMiMC7([low, next], 0) with its round values, the exclusion path,
//            exclusion_root: 66 permutations
//   warp 2   the low, next, gap_lo and gap_hi bits, then labeled_change_witness (7 permutations)
// The warps write disjoint variables, so no barrier is needed.
__global__ void __launch_bounds__(96) k_labeled_witness(LabeledLayout L, uint32_t w_stride, LabeledInputs in, uint32_t batch,
                                                        Fr* __restrict__ W, int* flag) {
    const uint32_t role = threadIdx.x >> 5;
    const uint32_t p = blockIdx.x * 32 + (threadIdx.x & 31);
    if (p >= batch) return;
    Fr* w = W + (uint64_t)p * w_stride;
    if (role == 0) {
        labeled_note_witness(L, w, in, p, flag);
    } else if (role == 1) {
        const Fr lo = fr_from_u64(in.low[p]), nx = fr_from_u64(in.next[p]);
        w[15] = lo; w[16] = nx;
        const Fr leaf = mimc7_hash2<true>(lo, nx, w + L.xleaf_base, w + L.xleaf_base + L.perm);
        w[L.xleaf_out] = leaf;
        w[4] = witness_path(leaf, w + L.excl_base, L.depth, L.lvl_size, L.perm, in.excl_siblings + 32ull * L.depth * p,
                            in.excl_path_bits[p], flag);
    } else {
        // x = label + 1 <= 2^32
        const uint64_t lo = in.low[p], nx = in.next[p], x = (uint64_t)in.labels[p] + 1;
        store_range_bits(w + L.low_bits, lo);
        store_range_bits(w + L.next_bits, nx);
        store_range_bits(w + L.gap_lo_bits, gap_bits(x, lo));
        store_range_bits(w + L.gap_hi_bits, gap_bits(nx, x));
        labeled_change_witness(L, w, in, p, flag);
    }
}

// Witness of the labeled association withdraw statement, layout of DESIGN.md section 3
// (== oracle/labeled_association_circuit.py); row p starts at W + p * w_stride, Montgomery form.  The labeled kernel's shape:
// a CTA covers 32 proofs with three warps, one per independent chain of a proof, writing disjoint variables without a barrier:
//   warp 0   labeled_note_witness: 70 permutations at depth 32, the critical path
//   warp 1   assoc_leaf = label + 1, the association path from it, association_root: 64 permutations
//   warp 2   labeled_change_witness: 7 permutations and the range bits
__global__ void __launch_bounds__(96) k_labeled_association_witness(LabeledAssociationLayout L, uint32_t w_stride, LabeledAssociationInputs in,
                                                                    uint32_t batch, Fr* __restrict__ W, int* flag) {
    const uint32_t role = threadIdx.x >> 5;
    const uint32_t p = blockIdx.x * 32 + (threadIdx.x & 31);
    if (p >= batch) return;
    Fr* w = W + (uint64_t)p * w_stride;
    if (role == 0) {
        labeled_note_witness(L, w, in, p, flag);
    } else if (role == 1) {
        const Fr leaf = fr_from_u64((uint64_t)in.labels[p] + 1);
        w[15] = leaf;
        w[4] = witness_path(leaf, w + L.assoc_base, L.depth, L.lvl_size, L.perm, in.assoc_siblings + 32ull * L.depth * p,
                            in.assoc_path_bits[p], flag);
    } else {
        labeled_change_witness(L, w, in, p, flag);
    }
}

// An owned note block's first variable (an input's spend key, an output's owner), blinding, amount (< 2^64), its 64 bits and
// the commitment MultiMiMC7([owner, blinding, token, amount], 4) with every round value, written into the block v.  Returns
// the commitment.
__device__ __forceinline__ Fr owned_note(const OwnedTransferLayout& L, Fr* v, const Fr& first, const Fr& owner, const Fr& bl,
                                         const Fr& token, uint64_t amount, uint32_t cm, uint32_t cm_out) {
    const Fr one = Fr::one(), zero = Fr::zero();
    const Fr am = fr_from_u64(amount);
    v[0] = first; v[1] = bl; v[2] = am;
#pragma unroll 8
    for (uint32_t k = 0; k < TRANSFER_AMOUNT_BITS; k++) v[3 + k] = ((amount >> k) & 1) ? one : zero;
    const Fr xs[4] = {owner, bl, token, am};
    const Fr r = mimc7_multi_hash<true>(xs, Fr::from_u32(OWNED_COMMITMENT_KEY), v + cm, L.perm);
    v[cm_out] = r;
    return r;
}

// Witness of the owned transfer statement, layout of DESIGN.md section 3 (== oracle/owned_circuit.py); row p starts at
// W + p * w_stride, Montgomery form.  The transfer kernel's shape: a CTA covers 32 proofs with four warps, one per
// independent hash chain of a proof, so no warp diverges and a proof's critical path is one input's owner, commitment and
// Merkle path (5 + 2 * depth permutations):
//   warps 0, 1   input i: the owner with its round values, amount bits, commitment, the depth levels
//   warps 2, 3   input j - 2's owner and commitment again in registers (no stores), its nullifier with its round values,
//                then output j - 2: amount bits, commitment (12 permutations)
// After the barrier, warp 0 writes the proof's remaining scalars (public amount, recipient, nf_diff_inv).  Only the low
// `depth` bits of a path word count, in the levels and in the nullifier's index alike.
__global__ void __launch_bounds__(128) k_owned_transfer_witness(OwnedTransferLayout L, uint32_t w_stride, OwnedTransferInputs in,
                                                                uint32_t batch, Fr* __restrict__ W, int* flag) {
    const uint32_t role = threadIdx.x >> 5;
    const uint32_t p = blockIdx.x * 32 + (threadIdx.x & 31);
    const bool active = p < batch;
    Fr* w = W + (uint64_t)p * w_stride;
    const Fr one = Fr::one();
    if (active) {
        const Fr token = load_canonical<Fr>(in.tokens + 32ull * p, flag);
        const Fr k3 = Fr::from_u32(OWNED_OWNER_KEY);
        const uint32_t i = role & 1;
        Fr* v = w + L.inp(i);
        const Fr s = load_canonical<Fr>(in.in_keys + 64ull * p + 32 * i, flag);
        const Fr bl = load_canonical<Fr>(in.in_blindings + 64ull * p + 32 * i, flag);
        const uint64_t amount = in.in_amounts[2ull * p + i];
        const uint32_t bits = in.in_bits[2ull * p + i];
        if (role < 2) {
            const Fr s1[1] = {s};
            const Fr owner = mimc7_multi_hash<true>(s1, k3, v + L.owner_perm, L.perm);
            const Fr cm = owned_note(L, v, s, owner, bl, token, amount, L.in_cm, L.in_cm_out);
            witness_path(cm, v + L.lvl_base, L.depth, L.lvl_size, L.perm, in.in_sib + 32ull * L.depth * (2ull * p + i), bits, flag);
        } else {
            const Fr s1[1] = {s};
            const Fr owner = mimc7_multi_hash<false>(s1, k3, nullptr, 0);
            const Fr note[4] = {owner, bl, token, fr_from_u64(amount)};
            const Fr cm = mimc7_multi_hash<false>(note, Fr::from_u32(OWNED_COMMITMENT_KEY), nullptr, 0);
            const uint32_t mask = L.depth >= 32 ? 0xffffffffu : (1u << L.depth) - 1;
            const Fr nf_in[3] = {s, cm, Fr::from_u32(bits & mask)};
            w[5 + i] = mimc7_multi_hash<true>(nf_in, Fr::from_u32(OWNED_NULLIFIER_KEY), v + L.nf_perm, L.perm);
            Fr* o = w + L.out(i);
            const Fr oo = load_canonical<Fr>(in.out_owners + 64ull * p + 32 * i, flag);
            const Fr ob = load_canonical<Fr>(in.out_blindings + 64ull * p + 32 * i, flag);
            w[7 + i] = owned_note(L, o, oo, oo, ob, token, in.out_amounts[2ull * p + i], L.out_cm, L.out_cm_out);
        }
        if (role == 0) {
            Fr re = load_canonical<Fr>(in.recipients + 32ull * p, flag);
            w[0] = one;
            w[1] = load_canonical<Fr>(in.roots + 32ull * p, flag);
            w[3] = token; w[4] = re;
            w[9] = re.sqr();
        }
    }
    __syncthreads();   // warps 1..3 wrote the amounts and nullifiers read below
    if (active && role == 0) {
        Fr a_in = w[L.inp(0) + 2] + w[L.inp(1) + 2], a_out = w[L.out(0) + 2] + w[L.out(1) + 2];
        w[2] = a_out - a_in;
        w[10] = (w[5] - w[6]).inv();   // inv(0) = 0: two inputs with one nullifier leave the row unsatisfiable
    }
}

// An owned labeled note block's first variable (an input's spend key, an output's owner), blinding, amount (< 2^64), its 64
// bits, and the precommitment and the leaf with every round value, their rounds from v + n + L.pre and v + n + L.leaf.
// Returns the leaf.
__device__ __forceinline__ Fr owned_labeled_note(const OwnedLabeledTransferLayout& L, Fr* v, uint32_t n, const Fr& first, const Fr& owner,
                                                 const Fr& bl, const Fr& token, uint64_t amount, const Fr& label) {
    const Fr one = Fr::one(), zero = Fr::zero();
    const Fr am = fr_from_u64(amount);
    v[0] = first; v[1] = bl; v[2] = am;
#pragma unroll 8
    for (uint32_t k = 0; k < LABELED_AMOUNT_BITS; k++) v[3 + k] = ((amount >> k) & 1) ? one : zero;
    const Fr pre_in[2] = {owner, bl};
    const Fr pre = mimc7_multi_hash<true>(pre_in, Fr::from_u32(OWNED_LABELED_PRE_KEY), v + n + L.pre, L.perm);
    v[n + L.pre_out] = pre;
    const Fr leaf_in[4] = {pre, token, am, label};
    const Fr leaf = mimc7_multi_hash<true>(leaf_in, Fr::from_u32(OWNED_LABELED_LEAF_KEY), v + n + L.leaf, L.perm);
    v[n + L.leaf_out] = leaf;
    return leaf;
}

// Witness of the owned labeled transfer statement, layout of DESIGN.md section 3 (== oracle/owned_labeled_circuit.py); row p
// starts at W + p * w_stride, Montgomery form.  The owned transfer kernel's split plus a fifth warp for the association path:
// a CTA covers 32 proofs with five warps, one per independent hash chain of a proof, so no warp diverges and a proof's
// critical path is one input's owner, precommitment, leaf and pool path (7 + 2 * depth permutations):
//   warps 0, 1   input i: the owner with its round values, amount bits, precommitment, leaf, the depth pool levels
//   warps 2, 3   input j - 2's owner, precommitment and leaf again in registers (no stores), its nullifier with its round
//                values, then output j - 2: amount bits, precommitment, leaf (16 permutations)
//   warp 4       the scalars, the label and withdrawn bits, assoc_leaf = label + 1 and the association path (2 * depth)
// After the barrier, warp 0 writes nf_diff_inv.  Only the low `depth` bits of a path word count, in the levels and in the
// nullifier's index alike.
__global__ void __launch_bounds__(160) k_owned_labeled_transfer_witness(OwnedLabeledTransferLayout L, uint32_t w_stride,
                                                                        OwnedLabeledTransferInputs in, uint32_t batch, Fr* __restrict__ W,
                                                                        int* flag) {
    const uint32_t role = threadIdx.x >> 5;
    const uint32_t p = blockIdx.x * 32 + (threadIdx.x & 31);
    const bool active = p < batch;
    Fr* w = W + (uint64_t)p * w_stride;
    if (active) {
        const Fr token = load_canonical<Fr>(in.tokens + 32ull * p, flag);
        const uint32_t label = in.labels[p];
        const Fr la = Fr::from_u32(label);
        if (role < 4) {
            const Fr k3 = Fr::from_u32(OWNED_OWNER_KEY);
            const uint32_t i = role & 1;
            Fr* v = w + L.inp(i);
            const Fr s = load_canonical<Fr>(in.in_keys + 64ull * p + 32 * i, flag);
            const Fr bl = load_canonical<Fr>(in.in_blindings + 64ull * p + 32 * i, flag);
            const uint64_t amount = in.in_amounts[2ull * p + i];
            const uint32_t bits = in.in_bits[2ull * p + i];
            const Fr s1[1] = {s};
            if (role < 2) {
                const Fr owner = mimc7_multi_hash<true>(s1, k3, v + L.owner_perm, L.perm);
                const Fr leaf = owned_labeled_note(L, v, L.perm, s, owner, bl, token, amount, la);
                witness_path(leaf, v + L.lvl_base, L.depth, L.lvl_size, L.perm, in.in_sib + 32ull * L.depth * (2ull * p + i), bits, flag);
            } else {
                const Fr owner = mimc7_multi_hash<false>(s1, k3, nullptr, 0);
                const Fr pre_in[2] = {owner, bl};
                const Fr pre = mimc7_multi_hash<false>(pre_in, Fr::from_u32(OWNED_LABELED_PRE_KEY), nullptr, 0);
                const Fr leaf_in[4] = {pre, token, fr_from_u64(amount), la};
                const Fr leaf = mimc7_multi_hash<false>(leaf_in, Fr::from_u32(OWNED_LABELED_LEAF_KEY), nullptr, 0);
                const uint32_t mask = L.depth >= 32 ? 0xffffffffu : (1u << L.depth) - 1;
                const Fr nf_in[3] = {s, leaf, Fr::from_u32(bits & mask)};
                w[6 + i] = mimc7_multi_hash<true>(nf_in, Fr::from_u32(OWNED_NULLIFIER_KEY), v + L.nf_perm, L.perm);
                Fr* o = w + L.out(i);
                const Fr oo = load_canonical<Fr>(in.out_owners + 64ull * p + 32 * i, flag);
                const Fr ob = load_canonical<Fr>(in.out_blindings + 64ull * p + 32 * i, flag);
                w[8 + i] = owned_labeled_note(L, o, 0, oo, oo, ob, token, in.out_amounts[2ull * p + i], la);
            }
        } else {
            const Fr one = Fr::one();
            const Fr re = load_canonical<Fr>(in.recipients + 32ull * p, flag);
            const uint64_t wd = in.withdrawn[p];
            w[0] = one;
            w[1] = load_canonical<Fr>(in.roots + 32ull * p, flag);
            w[3] = token; w[4] = fr_from_u64(wd); w[5] = re;
            w[10] = re.sqr();
            w[12] = la;
            store_range_bits(w + L.label_bits, label, LABELED_LABEL_BITS);
            store_range_bits(w + L.withdrawn_bits, wd, LABELED_AMOUNT_BITS);
            const Fr aleaf = fr_from_u64((uint64_t)label + 1);
            w[13] = aleaf;
            w[2] = witness_path(aleaf, w + L.assoc_base, L.depth, L.lvl_size, L.perm, in.assoc_sib + 32ull * L.depth * p,
                                in.assoc_bits[p], flag);
        }
    }
    __syncthreads();   // warps 2 and 3 wrote the nullifiers read below
    if (active && role == 0) w[11] = (w[6] - w[7]).inv();   // inv(0) = 0: two inputs with one nullifier leave the row unsatisfiable
}

// Witness of the ragequit statement, layout of DESIGN.md section 3 (== oracle/ragequit_circuit.py); row p starts at
// W + p * w_stride, Montgomery form.  A CTA covers 32 proofs with two warps, one per independent hash chain of a proof, so no
// warp diverges and a proof's critical path is the owner, precommitment, leaf and pool path (7 + 2 * depth permutations):
//   warp 0   the spend key and blinding, the owner with its round values, the precommitment, the leaf, the depth pool levels
//   warp 1   the owner, precommitment and leaf again in registers (no stores), the nullifier with its round values, and the
//            scalars (ONE, root, token, amount, label, recipient, recipient_sq)
// No warp reads what another wrote, so there is no barrier.  Only the low `depth` bits of the path word count, in the levels
// and in the nullifier's index alike.
__global__ void __launch_bounds__(64) k_ragequit_witness(RagequitLayout L, uint32_t w_stride, RagequitInputs in, uint32_t batch,
                                                         Fr* __restrict__ W, int* flag) {
    const uint32_t p = blockIdx.x * 32 + (threadIdx.x & 31);
    if (p >= batch) return;
    Fr* w = W + (uint64_t)p * w_stride;
    const Fr token = load_canonical<Fr>(in.tokens + 32ull * p, flag);
    const Fr am = fr_from_u64(in.amounts[p]);
    const Fr la = Fr::from_u32(in.labels[p]);
    const Fr s = load_canonical<Fr>(in.spend_keys + 32ull * p, flag);
    const Fr bl = load_canonical<Fr>(in.blindings + 32ull * p, flag);
    const uint32_t bits = in.path_bits[p];
    const Fr s1[1] = {s};
    const Fr k3 = Fr::from_u32(OWNED_OWNER_KEY), k6 = Fr::from_u32(OWNED_LABELED_PRE_KEY), k7 = Fr::from_u32(OWNED_LABELED_LEAF_KEY);
    if (threadIdx.x < 32) {
        w[8] = s; w[9] = bl;
        const Fr owner = mimc7_multi_hash<true>(s1, k3, w + L.owner_perm, L.perm);
        const Fr pre_in[2] = {owner, bl};
        const Fr pre = mimc7_multi_hash<true>(pre_in, k6, w + L.pre, L.perm);
        w[L.pre_out] = pre;
        const Fr leaf_in[4] = {pre, token, am, la};
        const Fr leaf = mimc7_multi_hash<true>(leaf_in, k7, w + L.leaf, L.perm);
        w[L.leaf_out] = leaf;
        witness_path(leaf, w + L.lvl_base, L.depth, L.lvl_size, L.perm, in.siblings + 32ull * L.depth * p, bits, flag);
    } else {
        const Fr owner = mimc7_multi_hash<false>(s1, k3, nullptr, 0);
        const Fr pre_in[2] = {owner, bl};
        const Fr pre = mimc7_multi_hash<false>(pre_in, k6, nullptr, 0);
        const Fr leaf_in[4] = {pre, token, am, la};
        const Fr leaf = mimc7_multi_hash<false>(leaf_in, k7, nullptr, 0);
        const uint32_t mask = L.depth >= 32 ? 0xffffffffu : (1u << L.depth) - 1;
        const Fr nf_in[3] = {s, leaf, Fr::from_u32(bits & mask)};
        w[6] = mimc7_multi_hash<true>(nf_in, Fr::from_u32(OWNED_NULLIFIER_KEY), w + L.nf_perm, L.perm);
        const Fr re = load_canonical<Fr>(in.recipients + 32ull * p, flag);
        w[0] = Fr::one();
        w[1] = load_canonical<Fr>(in.roots + 32ull * p, flag);
        w[2] = token; w[3] = am; w[4] = la; w[5] = re;
        w[7] = re.sqr();
    }
}

// ---- host side ------------------------------------------------------------------------------------
void mimc_constants_host(Fr* out91) { mimc7_round_constants(out91); }

int32_t mimc_init(og_ctx* ctx) {
    Fr c[MIMC_ROUNDS];
    mimc7_round_constants(c);
    OG_CUDA(ctx, cudaMemcpyToSymbol(c_mimc, c, sizeof(c)));
    return OG_OK;
}

int32_t mimc_hash2_dev(og_ctx* ctx, const uint8_t* d_l, const uint8_t* d_r, uint64_t n, uint8_t* d_out) {
    if (n == 0) return OG_OK;
    OG_LAUNCH(ctx, k_hash2, (unsigned)((n + 63) / 64), 64, 0, d_l, d_r, n, d_out, ctx->d_flag);
    return OG_OK;
}

int32_t mimc_merkle_paths_dev(og_ctx* ctx, const uint8_t* d_leaves, const uint8_t* d_siblings, const uint32_t* d_bits,
                              uint32_t n_paths, uint32_t depth, uint8_t* d_out) {
    if (n_paths == 0) return OG_OK;
    OG_LAUNCH(ctx, k_merkle_paths, (n_paths + 31) / 32, 32, 0, d_leaves, d_siblings, d_bits, n_paths, depth, d_out, ctx->d_flag);
    return OG_OK;
}

int32_t mimc_to_mont_dev(og_ctx* ctx, const uint8_t* d_in, uint64_t n, Fr* d_out) {
    if (n == 0) return OG_OK;
    OG_LAUNCH(ctx, k_to_mont, (unsigned)((n + 127) / 128), 128, 0, d_in, n, d_out, ctx->d_flag);
    return OG_OK;
}
int32_t mimc_from_mont_dev(og_ctx* ctx, const Fr* d_in, uint64_t n, uint8_t* d_out) {
    if (n == 0) return OG_OK;
    OG_LAUNCH(ctx, k_from_mont, (unsigned)((n + 127) / 128), 128, 0, d_in, n, d_out);
    return OG_OK;
}

template <NoteHash H>
static int32_t note_hash_launch(og_ctx* ctx, const StatementInputs& cols, uint64_t n, uint8_t* d_out) {
    OG_LAUNCHN(ctx, NOTE_HASHES[H].name, k_note_hash<H>, (unsigned)((n + 63) / 64), 64, 0, cols, n, d_out, ctx->d_flag);
    return OG_OK;
}

template <size_t... H>
static int32_t note_hash_dispatch(og_ctx* ctx, NoteHash h, const StatementInputs& cols, uint64_t n, uint8_t* d_out,
                                  std::index_sequence<H...>) {
    static constexpr int32_t (*launch[])(og_ctx*, const StatementInputs&, uint64_t, uint8_t*) = {note_hash_launch<NoteHash(H)>...};
    return launch[h](ctx, cols, n, d_out);
}

int32_t note_hash_dev(og_ctx* ctx, NoteHash h, const StatementInputs& cols, uint64_t n, uint8_t* d_out) {
    if (n == 0) return OG_OK;
    return note_hash_dispatch(ctx, h, cols, n, d_out, std::make_index_sequence<std::size(NOTE_HASHES)>{});
}

// levels: Montgomery-form buffer holding n + n/2 + ... + 1 elements, level 0 already filled
int32_t mimc_tree_build_dev(og_ctx* ctx, Fr* d_levels, uint64_t n_leaves) {
    Fr* in = d_levels;
    for (uint64_t n = n_leaves; n > 1; n >>= 1) {
        Fr* out = in + n;
        OG_LAUNCH(ctx, k_tree_level, (unsigned)((n / 2 + 63) / 64), 64, 0, in, n / 2, out);
        in = out;
    }
    return OG_OK;
}

// d_nodes: Montgomery buffer, level 0 (the n new leaves) already filled; levels 1..depth are appended behind it.
// h_aux (host): 2*depth Montgomery elements = left boundary per level, then empty-subtree root per level (kernel arguments).
int32_t mimc_tree_append_dev(og_ctx* ctx, uint32_t depth, uint64_t start, uint64_t n, const Fr* h_aux, Fr* d_nodes) {
    Fr* in = d_nodes;
    uint64_t c0 = start, n_in = n;
    for (uint32_t l = 0; l < depth; l++) {
        uint64_t p0 = c0 >> 1, p1 = (c0 + n_in - 1) >> 1, n_out = p1 - p0 + 1;
        Fr* out = in + n_in;
        OG_LAUNCH(ctx, k_tree_append_level, (unsigned)((n_out + 63) / 64), 64, 0, in, c0, n_in, p0, n_out, h_aux[l], h_aux[depth + l], out);
        in = out; c0 = p0; n_in = n_out;
    }
    return OG_OK;
}

// One CTA covers 32 proofs in every statement's kernel; the transfer, association, exclusion, labeled, labeled association,
// owned transfer, owned labeled transfer and ragequit kernels give a proof more than one warp.
int32_t statement_witness_dev(og_ctx* ctx, Statement s, uint32_t depth, uint32_t w_stride, const StatementInputs& in, uint32_t batch,
                              Fr* d_W) {
    if (batch == 0) return OG_OK;
    if (w_stride < STATEMENTS[s].shape(depth).n_vars) return OG_E_INVALID;
    const uint8_t* const* a = in.p;
    const uint32_t grid = (batch + 31) / 32;
    switch (s) {
    case ST_WITHDRAW:
        OG_LAUNCH(ctx, k_withdraw_witness, grid, 32, 0, WithdrawLayout::make(depth), w_stride, a[0], a[1], a[2], a[3],
                  (const uint32_t*)a[4], batch, d_W, ctx->d_flag);
        break;
    case ST_DEPOSIT:
        OG_LAUNCH(ctx, k_deposit_witness, grid, 32, 0, DepositLayout::make(), w_stride, a[0], a[1], a[2], batch, d_W, ctx->d_flag);
        break;
    case ST_TRANSFER: {
        const TransferInputs t{a[0], a[1], a[2], a[3], a[4], (const uint64_t*)a[5], a[6], (const uint32_t*)a[7], a[8], a[9],
                               (const uint64_t*)a[10]};
        OG_LAUNCH(ctx, k_transfer_witness, grid, 128, 0, TransferLayout::make(depth), w_stride, t, batch, d_W, ctx->d_flag);
        break;
    }
    case ST_ASSOCIATION: {
        const AssociationInputs t{a[0], a[1], a[2], a[3], (const uint32_t*)a[4], a[5], (const uint32_t*)a[6]};
        OG_LAUNCH(ctx, k_association_witness, grid, 64, 0, AssociationLayout::make(depth), w_stride, t, batch, d_W, ctx->d_flag);
        break;
    }
    case ST_EXCLUSION: {
        const ExclusionInputs t{a[0], a[1], a[2], a[3], (const uint32_t*)a[4], (const uint64_t*)a[5], (const uint64_t*)a[6], a[7],
                                (const uint32_t*)a[8]};
        OG_LAUNCH(ctx, k_exclusion_witness, grid, 64, 0, ExclusionLayout::make(depth), w_stride, t, batch, d_W, ctx->d_flag);
        break;
    }
    case ST_LABELED: {
        const LabeledInputs t{a[0], a[1], (const uint64_t*)a[2], a[3], a[4], (const uint64_t*)a[5], (const uint32_t*)a[6], a[7],
                              (const uint32_t*)a[8], a[9], a[10], (const uint64_t*)a[11], (const uint64_t*)a[12], a[13],
                              (const uint32_t*)a[14]};
        OG_LAUNCH(ctx, k_labeled_witness, grid, 96, 0, LabeledLayout::make(depth), w_stride, t, batch, d_W, ctx->d_flag);
        break;
    }
    case ST_LABELED_ASSOCIATION: {
        const LabeledAssociationInputs t{a[0], a[1], (const uint64_t*)a[2], a[3], a[4], (const uint64_t*)a[5], (const uint32_t*)a[6], a[7],
                                         (const uint32_t*)a[8], a[9], a[10], a[11], (const uint32_t*)a[12]};
        OG_LAUNCH(ctx, k_labeled_association_witness, grid, 96, 0, LabeledAssociationLayout::make(depth), w_stride, t, batch, d_W,
                  ctx->d_flag);
        break;
    }
    case ST_OWNED_TRANSFER: {
        const OwnedTransferInputs t{a[0], a[1], a[2], a[3], a[4], (const uint64_t*)a[5], a[6], (const uint32_t*)a[7], a[8], a[9],
                                    (const uint64_t*)a[10]};
        OG_LAUNCH(ctx, k_owned_transfer_witness, grid, 128, 0, OwnedTransferLayout::make(depth), w_stride, t, batch, d_W, ctx->d_flag);
        break;
    }
    case ST_OWNED_LABELED_TRANSFER: {
        const OwnedLabeledTransferInputs t{a[0], a[1], a[2], (const uint64_t*)a[3], (const uint32_t*)a[4], a[5], a[6], (const uint64_t*)a[7],
                                           a[8], (const uint32_t*)a[9], a[10], a[11], (const uint64_t*)a[12], a[13], (const uint32_t*)a[14]};
        OG_LAUNCH(ctx, k_owned_labeled_transfer_witness, grid, 160, 0, OwnedLabeledTransferLayout::make(depth), w_stride, t, batch, d_W,
                  ctx->d_flag);
        break;
    }
    case ST_RAGEQUIT: {
        const RagequitInputs t{a[0], a[1], a[2], (const uint64_t*)a[3], (const uint32_t*)a[4], a[5], a[6], a[7], (const uint32_t*)a[8]};
        OG_LAUNCH(ctx, k_ragequit_witness, grid, 64, 0, RagequitLayout::make(depth), w_stride, t, batch, d_W, ctx->d_flag);
        break;
    }
    }
    return OG_OK;
}

}  // namespace og

#include "bjj_impl.cuh"
#include "note_impl.cuh"
