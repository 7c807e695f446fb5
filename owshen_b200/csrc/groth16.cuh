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
// true iff the key has the deposit statement's shape (n_vars, n_pub, n_constraints): its layout is fixed, so the shape identifies it
bool pk_is_deposit(const og_pk* pk);
// window bits of the A (G1), B (G2) and C' (G1) MSMs the key was loaded with
void pk_window_bits(const og_pk* pk, uint32_t* c3);
int32_t prove_withdraw_dev(og_ctx* ctx, const og_pk* pk, const uint8_t* d_null, const uint8_t* d_sec, const uint8_t* d_rec,
                           const uint8_t* d_sib, const uint32_t* d_bits, uint32_t batch, const uint8_t* d_rs, uint8_t* d_proofs,
                           uint8_t* d_public);
int32_t prove_deposit_dev(og_ctx* ctx, const og_pk* pk, const uint8_t* d_null, const uint8_t* d_sec, const uint8_t* d_dep, uint32_t batch,
                          const uint8_t* d_rs, uint8_t* d_proofs, uint8_t* d_public);
// the depth d in 1..32 whose transfer layout matches the key's n_vars, n_constraints and n_pub = 8; 0 = not a transfer key
uint32_t pk_transfer_depth(const og_pk* pk);
int32_t prove_transfer_dev(og_ctx* ctx, const og_pk* pk, const TransferInputs& in, uint32_t batch, const uint8_t* d_rs, uint8_t* d_proofs,
                           uint8_t* d_public);
// the chunk size and lanes prove_batch uses for `batch` proofs with this key, and the scratch bytes of one lane
void pk_prover_plan(const og_pk* pk, uint32_t batch, uint32_t* chunk, uint32_t* lanes, uint64_t* scratch_bytes_per_lane);
int32_t prove_witness_dev(og_ctx* ctx, const og_pk* pk, const uint8_t* d_wit, uint32_t batch, const uint8_t* d_rs, uint8_t* d_proofs);
int32_t h_evals_dev(og_ctx* ctx, const og_pk* pk, const uint8_t* d_wit, uint8_t* d_out);
int32_t withdraw_witness_bytes_dev(og_ctx* ctx, uint32_t depth, const uint8_t* d_null, const uint8_t* d_sec, const uint8_t* d_rec,
                                   const uint8_t* d_sib, const uint32_t* d_bits, uint32_t batch, uint8_t* d_out);
int32_t deposit_witness_bytes_dev(og_ctx* ctx, const uint8_t* d_null, const uint8_t* d_sec, const uint8_t* d_dep, uint32_t batch,
                                  uint8_t* d_out);
int32_t transfer_witness_bytes_dev(og_ctx* ctx, uint32_t depth, const TransferInputs& in, uint32_t batch, uint8_t* d_out);
// setup.cu
int32_t setup_withdraw(og_ctx* ctx, uint32_t depth, const uint8_t* toxic160, uint8_t* pk_out, uint64_t* pk_len,
                       uint8_t* vk_out, uint64_t* vk_len);
// the caller's R1CS: matrices A, B, C as CSR (row_ptr[3], col[3], coeffs[3]), validated before any work
int32_t setup_generic(og_ctx* ctx, uint32_t n_constraints, uint32_t n_vars, uint32_t n_pub, const uint32_t* const row_ptr[3],
                      const uint32_t* const col[3], const uint8_t* const coeffs[3], const uint8_t* toxic160, uint8_t* pk_out,
                      uint64_t* pk_len, uint8_t* vk_out, uint64_t* vk_len);
// pairing.cpp
int32_t groth16_verify_host(const uint8_t* vk, uint64_t vk_len, const uint8_t* pub, uint32_t n_pub, const uint8_t* proof);
}  // namespace og
