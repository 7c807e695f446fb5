// owshen_b200/csrc/msm.cuh -- interface of the bucket-method (Pippenger) MSM engine shared by the
// one-shot MSM entry points (og_msm_g1/g2) and the batched Groth16 prover.
#pragma once
#include "common.cuh"

namespace og {

// How scalars are cut into signed c-bit digits and where each (digit, point) pair goes.
//   key   = (problem * key_stride_problem + window * key_stride_window) * nb + (|digit| - 1)
//   entry = ((index + window * tidx_window_stride) << 1) | (digit < 0)
// One-shot MSM:   groups are windows  (key_stride_problem = 0, key_stride_window = 1, tidx stride 0).
// Batched prover: groups are proofs   (key_stride_problem = 1, key_stride_window = 0) and the table
//                 holds the precomputed multiples 2^(c*w) * P_i at index i + w * n_points.
struct DigitPlan {
    const uint32_t* scalars;     // 8 x u32 per scalar; canonical integers or Montgomery Fr
    uint64_t n;                  // scalars per problem
    uint64_t scalar_stride;      // elements between consecutive problems
    uint32_t n_problems;
    uint32_t c, n_windows, nb;   // nb = 2^(c-1) buckets per group
    uint32_t key_stride_problem, key_stride_window;
    uint32_t tidx_window_stride;
    int32_t montgomery;          // 1: scalars are Montgomery-form Fr and are converted on the fly
};

static inline uint32_t msm_windows(uint32_t c) { return (255 + c - 1) / c; }

// Fills counts[key], offsets[key] (exclusive scan; offsets[n_keys] = the total number of entries) and sorted[]: the entries
// of each bucket are contiguous, in no particular order.
// One-shot MSMs (key_stride_window != 0): d_cursor is n_keys u32 of scratch; d_stage and d_tiles are unused.
// Batched prover (key_stride_window == 0, key_stride_problem == 1, nb <= 2^15): a partitioned sort that needs
//   d_stage: msm_sort_stage_bytes(n_problems * n * n_windows) of staging and d_tiles: msm_sort_tile_bytes(n_problems, nb, n);
//   d_cursor is unused.
int32_t msm_sort_digits(og_ctx* ctx, const DigitPlan& plan, uint32_t n_keys, uint32_t* d_counts,
                        uint32_t* d_offsets /* n_keys + 1 */, uint32_t* d_cursor, uint32_t* d_sorted,
                        uint32_t* d_stage = nullptr, uint32_t* d_tiles = nullptr);
size_t msm_sort_stage_bytes(uint64_t n_entries);
size_t msm_sort_tile_bytes(uint32_t n_problems, uint32_t nb, uint64_t n);

// Accumulate every bucket and reduce each group to sum_b (b+1) * bucket_b.
// d_buckets: n_groups * nb XYZZ scratch; d_lvl: msm_lvl_elems(n_groups, nb) XYZZ scratch;
// d_heavy: 2 * n_keys + 4 u32 scratch; n_entries_max: upper bound on the sorted entries (sets the heavy-bucket cap);
// d_perm: n_keys u32 scratch (the sort's cursor array may be reused); result: d_totals[n_groups].
int32_t msm_buckets_g1(og_ctx* ctx, const G1Affine* d_table, const uint32_t* d_sorted, const uint32_t* d_offsets,
                       const uint32_t* d_counts, uint32_t n_groups, uint32_t nb, uint64_t n_entries_max, G1XYZZ* d_buckets,
                       G1XYZZ* d_lvl, uint32_t* d_heavy, uint32_t* d_perm, G1XYZZ* d_totals, void* aff_scratch = nullptr);
int32_t msm_buckets_g2(og_ctx* ctx, const G2Affine* d_table, const uint32_t* d_sorted, const uint32_t* d_offsets,
                       const uint32_t* d_counts, uint32_t n_groups, uint32_t nb, uint64_t n_entries_max, G2XYZZ* d_buckets,
                       G2XYZZ* d_lvl, uint32_t* d_heavy, uint32_t* d_perm, G2XYZZ* d_totals, void* aff_scratch = nullptr);
// aff_scratch: experiment builds only (-DOG_EXPERIMENT_AFFINE): non-null selects the rejected batched-affine accumulation
// (csrc/experiments/bucket_affine.cuh); the shipped library ignores it and the sizes are 0
size_t msm_aff_scratch_bytes_g1(uint64_t n_keys);
size_t msm_aff_scratch_bytes_g2(uint64_t n_keys);
static inline size_t msm_lvl_elems(uint32_t n_groups, uint32_t nb) { return 4 * ((size_t)n_groups * ((nb + 7) / 8) + 16); }   // RED_FAN = 8

// one-shot MSMs on device buffers holding boundary bytes (affine points, canonical scalars)
int32_t msm_g1_dev(og_ctx* ctx, const uint8_t* d_points, const uint8_t* d_scalars, uint64_t n, uint8_t* d_out64);
int32_t msm_g2_dev(og_ctx* ctx, const uint8_t* d_points, const uint8_t* d_scalars, uint64_t n, uint8_t* d_out128);
int32_t sum_g1_dev(og_ctx* ctx, const uint8_t* d_points, uint64_t n, uint8_t* d_out64);
int32_t sum_g2_dev(og_ctx* ctx, const uint8_t* d_points, uint64_t n, uint8_t* d_out128);

// boundary conversions for points
int32_t g1_bytes_to_mont(og_ctx* ctx, const uint8_t* d_in, uint64_t n, G1Affine* d_out);
int32_t g2_bytes_to_mont(og_ctx* ctx, const uint8_t* d_in, uint64_t n, G2Affine* d_out);
int32_t g1_mont_to_bytes(og_ctx* ctx, const G1Affine* d_in, uint64_t n, uint8_t* d_out);
int32_t g2_mont_to_bytes(og_ctx* ctx, const G2Affine* d_in, uint64_t n, uint8_t* d_out);

// fixed-base window tables: table[w * n + i] = 2^(c*w) * P_i  (w < n_windows), affine Montgomery.
// table[0..n) must already hold the points.
int32_t msm_build_table_g1(og_ctx* ctx, G1Affine* d_table, uint32_t n, uint32_t c, uint32_t n_windows);
int32_t msm_build_table_g2(og_ctx* ctx, G2Affine* d_table, uint32_t n, uint32_t c, uint32_t n_windows);

// out[i] = scalars[i] * generator (setup): scalars canonical bytes on device, out affine Montgomery
int32_t fixed_base_mul_g1(og_ctx* ctx, const uint8_t* d_scalars, uint64_t n, G1Affine* d_out);
int32_t fixed_base_mul_g2(og_ctx* ctx, const uint8_t* d_scalars, uint64_t n, G2Affine* d_out);

}  // namespace og
