// owshen_b200/csrc/groth16.cuh -- interface of the batched Groth16 prover, pk handling and setup.
#pragma once
#include "common.cuh"
#include "mimc.cuh"

struct og_pk;

namespace og {
int32_t pk_load(og_ctx* ctx, const uint8_t* bytes, uint64_t len, og_pk** out);
void pk_free(og_pk* pk);
// true iff the key's tables live on the device `ctx` runs on (a key is bound to the device of the ctx that loaded it)
bool pk_on_device_of(const og_pk* pk, const og_ctx* ctx);
void pk_info(const og_pk* pk, uint32_t* n_vars, uint32_t* n_pub, uint32_t* log_m, uint32_t* depth);
// window bits of the A (G1), B (G2) and C' (G1) MSMs the key was loaded with
void pk_window_bits(const og_pk* pk, uint32_t* c3);
// The depth the key proves statement s at, or -1 when it is not that statement's key.  A withdraw key records its depth
// (setup_withdraw, ptau_prepare_withdraw); every other statement's key is recognised by its shape (n_pub, n_vars,
// n_constraints): deposit's is fixed, transfer and association take the first depth in 1..32 whose layout matches.
int32_t statement_key_depth(const og_pk* pk, Statement s);
// a batch of statement s's proofs from its device inputs; OG_E_INVALID for another statement's key, whatever the batch
int32_t prove_statement_dev(og_ctx* ctx, const og_pk* pk, Statement s, const StatementInputs& in, uint32_t batch, const uint8_t* d_rs,
                            uint8_t* d_proofs, uint8_t* d_public);
// the chunk size and lanes prove_batch uses for `batch` proofs with this key, and the scratch bytes of one lane
void pk_prover_plan(const og_pk* pk, uint32_t batch, uint32_t* chunk, uint32_t* lanes, uint64_t* scratch_bytes_per_lane);
int32_t prove_witness_dev(og_ctx* ctx, const og_pk* pk, const uint8_t* d_wit, uint32_t batch, const uint8_t* d_rs, uint8_t* d_proofs);
int32_t h_evals_dev(og_ctx* ctx, const og_pk* pk, const uint8_t* d_wit, uint8_t* d_out);
// statement s's full witnesses at `depth` as canonical bytes, n_vars * 32 per proof
int32_t statement_witness_bytes_dev(og_ctx* ctx, Statement s, uint32_t depth, const StatementInputs& in, uint32_t batch, uint8_t* d_out);
// byte offsets of a serialized pk's sections (og_load_pk's layout); false if the header or a section is malformed
struct PkLayout {
    uint32_t depth, n_constraints, n_vars, n_pub, log_m;
    uint64_t alpha1, beta1, beta2, delta1, delta2, qa, qb1, qb2, ql, qh, csr;   // csr: the A and B matrices that end the key
};
bool pk_layout(const uint8_t* bytes, uint64_t len, PkLayout& L);
// setup.cu
struct R1cs;
// boundary bytes of every pk/vk element: G1 alpha, beta, delta, A (n_vars), B (n_vars), L (n_priv), IC (n_pub + 1), H (m);
// G2 beta, delta, gamma, B (n_vars)
struct KeyPoints {
    const uint8_t *alpha1, *beta1, *delta1, *qa, *qb1, *ql, *ic, *qh;
    const uint8_t *beta2, *delta2, *gamma2, *qb2;
};
void key_sizes(const R1cs& cs, uint64_t* pk_len, uint64_t* vk_len);
int32_t write_keys(const R1cs& cs, uint32_t depth, const KeyPoints& P, uint8_t* pk_out, uint64_t* pk_len, uint8_t* vk_out, uint64_t* vk_len);
// og_groth16_setup's validation of the caller's R1CS
int32_t load_r1cs(uint32_t n_constraints, uint32_t n_vars, uint32_t n_pub, const uint32_t* const row_ptr[3], const uint32_t* const col[3],
                  const uint8_t* const coeffs[3], R1cs& cs);
Fr host_root_of_unity(uint32_t log_n);   // 7^((r-1) / 2^log_n)
int32_t setup_withdraw(og_ctx* ctx, uint32_t depth, const uint8_t* toxic160, uint8_t* pk_out, uint64_t* pk_len,
                       uint8_t* vk_out, uint64_t* vk_len);
// the caller's R1CS: matrices A, B, C as CSR (row_ptr[3], col[3], coeffs[3]), validated before any work
int32_t setup_generic(og_ctx* ctx, uint32_t n_constraints, uint32_t n_vars, uint32_t n_pub, const uint32_t* const row_ptr[3],
                      const uint32_t* const col[3], const uint8_t* const coeffs[3], const uint8_t* toxic160, uint8_t* pk_out,
                      uint64_t* pk_len, uint8_t* vk_out, uint64_t* vk_len);
// pairing.cpp
int32_t groth16_verify_host(const uint8_t* vk, uint64_t vk_len, const uint8_t* pub, uint32_t n_pub, const uint8_t* proof);
bool pairing_product_is_one(const G1Affine* P, const G2Affine* Q, int n);
// canonical bytes -> a point on the curve (G2: and in the subgroup); infinity is (0, 0)
bool load_g1(G1Affine& p, const uint8_t* b);
bool load_g2(G2Affine& p, const uint8_t* b);
// ceremony.cu: the two-phase setup ceremony (DESIGN.md section 4b)
int32_t ptau_new(og_ctx* ctx, uint32_t log_max, uint8_t* out, uint64_t* out_len);
int32_t ptau_contribute(og_ctx* ctx, const uint8_t* acc, uint64_t acc_len, const uint8_t* secrets96, const uint8_t* nonces96,
                        uint8_t* acc_out, uint64_t* acc_out_len, uint8_t* rec_out, uint64_t* rec_len);
int32_t ptau_verify(og_ctx* ctx, const uint8_t* prev, uint64_t prev_len, const uint8_t* next, uint64_t next_len, const uint8_t* rec,
                    uint64_t rec_len);
int32_t ptau_prepare(og_ctx* ctx, const uint8_t* acc, uint64_t acc_len, const R1cs& cs, uint32_t depth, uint8_t* pk_out, uint64_t* pk_len,
                     uint8_t* vk_out, uint64_t* vk_len);
int32_t phase2_contribute(og_ctx* ctx, const uint8_t* pk, uint64_t pk_len, const uint8_t* vk, uint64_t vk_len, const uint8_t* d32,
                          const uint8_t* nonce32, uint8_t* pk_out, uint64_t* pk_out_len, uint8_t* vk_out, uint64_t* vk_out_len,
                          uint8_t* rec_out, uint64_t* rec_len);
int32_t phase2_verify(og_ctx* ctx, const uint8_t* pk0, uint64_t pk0_len, const uint8_t* vk0, uint64_t vk0_len, const uint8_t* pk1,
                      uint64_t pk1_len, const uint8_t* vk1, uint64_t vk1_len, const uint8_t* rec, uint64_t rec_len);
// kernel-level entry points exposed for tests: out_i = s_i * P_i (or s_0 * P_i when !per_point), and the iNTT of 2^log_m points
int32_t scale_points_dev(og_ctx* ctx, int g2, const uint8_t* d_points, const uint8_t* d_scalars, uint64_t n, int per_point, uint8_t* d_out);
int32_t intt_points_dev(og_ctx* ctx, int g2, uint8_t* d_points, uint32_t log_m);
}  // namespace og
