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

// The engine below is one set of function templates on the coordinate field F: Fq = G1, Fq2 = G2.  msm.cu is compiled once per
// curve and instantiates them for that curve's F only.

// Accumulate every bucket and reduce each group to sum_b (b+1) * bucket_b.
// d_buckets: n_groups * nb XYZZ scratch; d_lvl: msm_lvl_elems(n_groups, nb) XYZZ scratch;
// d_heavy: 2 * n_keys + 4 u32 scratch; n_entries_max: upper bound on the sorted entries (sets the heavy-bucket cap);
// d_perm: n_keys u32 scratch (the sort's cursor array may be reused); result: d_totals[n_groups].
// few_groups: the groups are the windows of a one-shot MSM (msm.cu section 5b); the prover's groups are proofs.
template <class F>
int32_t msm_buckets(og_ctx* ctx, const Affine<F>* d_table, const uint32_t* d_sorted, const uint32_t* d_offsets, const uint32_t* d_counts,
                    uint32_t n_groups, uint32_t nb, uint64_t n_entries_max, XYZZ<F>* d_buckets, XYZZ<F>* d_lvl, uint32_t* d_heavy,
                    uint32_t* d_perm, XYZZ<F>* d_totals, bool few_groups = false);
static inline size_t msm_lvl_elems(uint32_t n_groups, uint32_t nb) { return 4 * ((size_t)n_groups * ((nb + 7) / 8) + 16); }   // RED_FAN = 8
// Heavy buckets of msm_buckets, with avg = n_entries_max / n_keys: a list of more than cap = max(128, 4 avg) entries goes to
// k_bucket_heavy, cut into segments of seg = max(2048, 4 avg) entries whose sums are written into d_lvl.  Both values must fit 32 bits
// (avg < 2^30).  While avg < 512 the segment sums always fit d_lvl: a heavy list takes at most one segment per min(cap + 1, 1024) of
// its entries, so fewer than (avg + 1) n_keys / min(cap + 1, 1024) <= n_keys / 2 segments exist.  From avg = 512 on, cap == seg, so a
// list of cap + 1 entries takes two segments and the count can exceed msm_lvl_elems by up to about 3 n_keys / (8 avg) elements.  The
// MSM and prover callers stay far below avg = 512 (one-shot MSMs 16 to 32, the prover's A, B and C' MSMs about 25, 13 and 34).
static inline uint32_t msm_heavy_cap(uint64_t avg) { return (uint32_t)(4 * avg < 128 ? 128 : 4 * avg); }
static inline uint32_t msm_heavy_seg(uint64_t avg) { return (uint32_t)(4 * avg < 2048 ? 2048 : 4 * avg); }

// Test/debug probes behind og_msm_bucket_sums and og_field_probe_raw (not used by the product).
// msm_bucket_sums: msm_buckets (few_groups as given) on caller-given lists -- d_points: n_points affine boundary points;
// d_sorted / d_offsets / d_counts as msm_buckets reads them, with n_entries_max >= offsets[n_keys] and a heavy plan whose segment
// sums fit d_lvl (msm_heavy_cap / msm_heavy_seg above; og_msm_bucket_sums checks both); out: n_groups totals and, when
// d_out_buckets is not null, the n_keys accumulated buckets, as affine boundary points.
template <class F>
int32_t msm_bucket_sums(og_ctx* ctx, const uint8_t* d_points, uint32_t n_points, const uint32_t* d_sorted, const uint32_t* d_offsets,
                        const uint32_t* d_counts, uint32_t n_groups, uint32_t nb, uint64_t n_entries_max, bool few_groups,
                        uint8_t* d_out_totals, uint8_t* d_out_buckets);
// field_probe_raw: raw Montgomery limbs in and out, no range check, through the functions the bucket kernels of each unit call
// (the probe kernels' own ptxas copies of them):
// G1 (Fq, 32 B) ops 0..3, G2 (Fq2, 64 B) ops 0..7 (msm.cu: k_field_probe_g1 / k_field_probe_g2)
template <class F> int32_t field_probe_raw(og_ctx* ctx, int32_t op, const uint8_t* d_a, const uint8_t* d_b, uint64_t n, uint8_t* d_out);

// one-shot MSM and plain sum on device buffers holding boundary bytes (affine points, canonical scalars); d_out: one affine point
template <class F> int32_t msm_dev(og_ctx* ctx, const uint8_t* d_points, const uint8_t* d_scalars, uint64_t n, uint8_t* d_out);
template <class F> int32_t sum_dev(og_ctx* ctx, const uint8_t* d_points, uint64_t n, uint8_t* d_out);

// boundary conversions for points
template <class F> int32_t points_bytes_to_mont(og_ctx* ctx, const uint8_t* d_in, uint64_t n, Affine<F>* d_out);
template <class F> int32_t points_mont_to_bytes(og_ctx* ctx, const Affine<F>* d_in, uint64_t n, uint8_t* d_out);

// fixed-base window tables: table[w * n + i] = 2^(c*w) * P_i  (w < n_windows), affine Montgomery.
// table[0..n) must already hold the points.
template <class F> int32_t msm_build_table(og_ctx* ctx, Affine<F>* d_table, uint32_t n, uint32_t c, uint32_t n_windows);

// out[i] = scalars[i] * generator (setup): scalars canonical bytes on device, out affine Montgomery
template <class F> int32_t fixed_base_mul(og_ctx* ctx, const uint8_t* d_scalars, uint64_t n, Affine<F>* d_out);

}  // namespace og
