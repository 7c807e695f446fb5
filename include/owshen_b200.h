/* include/owshen_b200.h -- C ABI of the H100-native (sm_90a) Groth16 backend (libowshen_b200.so).
 *
 * WHAT THIS REPLACES IN THE REFERENCE.  OwshenNetwork/owshen @ c7b1f00 has no prover, no FFI and no
 * plugin interface for proving (SURVEY.md section 0 / 8b), so there is no reference binding to cite
 * per entry point; this header DEFINES the boundary that BASELINE.json's north_star asks for
 * ("Rust prove()/verify()/MerkleTree ... through a thin C-ABI/FFI layer").  The conventions it
 * inherits from the reference are:
 *   - field elements: BN254 Fr, canonical little-endian 32 bytes
 *     (/root/reference/src/blockchain/tx/owshen_airdrop/babyjubjub/mod.rs:7-11);
 *   - fallible calls return a status instead of panicking, mirroring `anyhow::Result<T>`
 *     (/root/reference/src/blockchain/mod.rs:11); byte blobs are caller-owned buffers
 *     (the reference passes owned `Vec<u8>`, e.g. src/types/tx/custom.rs:258-287);
 *   - the natural call site is a service handler shaped like withdraw_handler
 *     (/root/reference/src/services/api_services/withdraw.rs:27-71); INTEGRATION.md shows the
 *     Rust `extern "C"` stub a maintainer would add there.
 *
 * Formats.  Fr / Fq: 32 B little-endian canonical (values >= modulus are rejected with
 * OG_E_ENCODING).  G1 affine: x || y (64 B).  G2 affine: x.c0 || x.c1 || y.c0 || y.c1 (128 B).
 * The point at infinity is the all-zero encoding.  Proof: A (G1) || B (G2) || C (G1) = 256 B.
 *
 * Threading.  An og_ctx owns one CUDA device and one stream; calls on one ctx must not overlap,
 * different ctxs are independent.  Host-pointer entry points copy H2D/D2H themselves and return
 * after the result is in the caller's buffer.  `_dev` entry points take DEVICE pointers, enqueue
 * on the ctx stream and return without synchronising (use og_sync / og_timer_*).
 *
 * There is NO CPU fallback: without a CUDA device og_init fails with OG_E_NO_DEVICE and nothing
 * else can be called (og_groth16_verify is a host function by design: three pairings).
 */
#ifndef OWSHEN_B200_H
#define OWSHEN_B200_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef struct og_ctx og_ctx;
typedef struct og_pk og_pk;

enum {
    OG_OK = 0,
    OG_E_INVALID = -1,     /* bad argument (null pointer, size out of range) */
    OG_E_ENCODING = -2,    /* non-canonical field element / malformed blob */
    OG_E_NO_DEVICE = -3,   /* no usable CUDA device: the library has no CPU path */
    OG_E_CUDA = -4,        /* a CUDA runtime call failed; see og_last_error */
    OG_E_NOMEM = -5,
    OG_E_VERIFY = -6       /* og_groth16_verify: well-formed proof that does not verify */
};

int32_t og_abi_version(void);
const char* og_strerror(int32_t code);
const char* og_last_error(const og_ctx* ctx);

/* ---- context ------------------------------------------------------------------------------- */
int32_t og_init(int32_t device, og_ctx** out);
void og_free(og_ctx* ctx);
int32_t og_sync(og_ctx* ctx);
/* the CUDA stream (cudaStream_t) every `_dev` entry point of ctx enqueues on: a host that orders other work against
 * the library without a host synchronisation (the NCCL all-gather of the sharded MSM) wraps it, e.g.
 * torch.cuda.ExternalStream(ptr) */
int32_t og_stream(og_ctx* ctx, void** out_cuda_stream);
/* CUDA-event timer on the ctx stream (bench.py times kernels with these, not torch events) */
int32_t og_timer_start(og_ctx* ctx);
int32_t og_timer_stop(og_ctx* ctx, float* ms);
/* number of this library's kernel launches enqueued on ctx since creation */
uint64_t og_launch_count(const og_ctx* ctx);
/* per-kernel timing: CUDA events around every launch while enabled; og_profile_dump synchronises and
 * writes "kernel,launches,total_ms" lines accumulated since the previous dump */
int32_t og_profile(og_ctx* ctx, int32_t enable);
int32_t og_profile_dump(og_ctx* ctx, char* buf, uint64_t cap);
/* integer-pipe micro-benchmark: achieved 32-bit multiply-add lane-ops per second */
int32_t og_imad_peak(og_ctx* ctx, double* mad_per_s, double* wide_mad_per_s);
/* same plus the rate of 32x32->64 multiply-adds issued as mad.lo.cc/madc.hi.cc carry chains (the shape of
 * a Montgomery row, IMAD.WIDE.U32.X): the honest roofline denominator of the field multiplier */
int32_t og_int_pipe_peaks(og_ctx* ctx, double* mad_per_s, double* wide_mad_per_s, double* carry_chain_wide_per_s);

/* SM cycles per dependent Fr multiply(+add) for one warp alone on a scheduler, and per iteration of two
 * independent chains: the latency that bounds the sequential MiMC chains (planning probe) */
int32_t og_mul_latency(og_ctx* ctx, double* cycles_dependent, double* cycles_two_chains);
/* planning probe for a hybrid multiplier: rates4 = {52x52-bit FP64-pipe products/s alone, 32x32-bit carry-chain
 * multiply-adds/s alone, and both rates when the two kinds run interleaved in every warp} */
int32_t og_hybrid_probe(og_ctx* ctx, double* rates4);
/* FP64 fused multiply-adds per second (planning probe: the FP64 pipe is idle in every kernel of this library) */
int32_t og_fp64_peak(og_ctx* ctx, double* dfma_per_s);

/* ---- element-wise field ops (parity probes for the limb arithmetic) ------------------------- */
/* field: 0 = Fq, 1 = Fr; op: 0 = mul, 1 = add, 2 = sub */
int32_t og_field_op(og_ctx* ctx, int32_t field, int32_t op, const uint8_t* a, const uint8_t* b,
                    uint64_t n, uint8_t* out);

/* ---- MiMC7 / Merkle (BASELINE config 2) ------------------------------------------------------ */
/* MiMC7 round constants as derived on the host (keccak chain from "mimc"): 91 * 32 B */
int32_t og_mimc7_constants(uint8_t* out, uint32_t* n_rounds);
/* out[i] = MultiMiMC7([left[i], right[i]], key = 0) */
int32_t og_mimc7_hash2(og_ctx* ctx, const uint8_t* left, const uint8_t* right, uint64_t n, uint8_t* out);
/* out_nodes: n_paths * (depth+1) * 32 B, node 0 = leaf ... node depth = root.
 * path_bits[p] bit l = 1: the running node is the RIGHT child at level l.  depth <= 32. */
int32_t og_mimc7_merkle_paths(og_ctx* ctx, const uint8_t* leaves, const uint8_t* siblings,
                              const uint32_t* path_bits, uint32_t n_paths, uint32_t depth,
                              uint8_t* out_nodes);
int32_t og_mimc7_merkle_paths_dev(og_ctx* ctx, const uint8_t* d_leaves, const uint8_t* d_siblings,
                                  const uint32_t* d_path_bits, uint32_t n_paths, uint32_t depth,
                                  uint8_t* d_out_nodes);
/* full tree build: levels[0] = leaves (n = 2^depth_built padded by the caller), returns all
 * levels concatenated: sum_{l=0..log2 n} (n >> l) * 32 B */
int32_t og_mimc7_merkle_build(og_ctx* ctx, const uint8_t* leaves, uint64_t n_leaves_pow2, uint8_t* out_levels);
/* append to a fixed-depth sparse tree (the incremental builder of SURVEY.md 8f.2): all nodes of levels 1..depth
 * touched by inserting n leaves at index `start`, in ONE call.  left_boundary[l] (32 B per level, l < depth) is the
 * stored node (l, (start >> l) - 1) when (start >> l) is odd (ignored otherwise); zeros[l] is the root of an empty
 * subtree of height l.  out_nodes: level 1 first, level l holds ((start+n-1)>>l) - (start>>l) + 1 nodes. */
int32_t og_mimc7_merkle_append(og_ctx* ctx, uint32_t depth, uint64_t start, const uint8_t* leaves, uint64_t n,
                               const uint8_t* left_boundary, const uint8_t* zeros, uint8_t* out_nodes);

/* ---- BabyJubJub EdDSA-style batch verification (SURVEY.md 8f.3) -------------------------------------------
 * Replaces a loop over PointCompressed::verify, /root/reference/src/blockchain/tx/owshen_airdrop/babyjubjub/
 * mod.rs:99-115 (with decompress :88-98, multiply :68-78, hash :202-204).  Per signature: pk_x 32 B and one
 * is_odd byte (PointCompressed, mod.rs:19), message 32 B, signature = R.x || R.y || s (96 B).
 * hash_kind 0 = the reference's placeholder product hash, 1 = MultiMiMC7 (not reference behaviour).
 * out_status[i]: 1 verifies, 0 does not, 2 = the reference would return Err (pk does not decompress). */
int32_t og_bjj_verify_batch(og_ctx* ctx, const uint8_t* pk_x, const uint8_t* pk_is_odd, const uint8_t* messages,
                            const uint8_t* signatures, uint32_t n, int32_t hash_kind, uint8_t* out_status);
int32_t og_bjj_verify_batch_dev(og_ctx* ctx, const uint8_t* d_pk_x, const uint8_t* d_pk_is_odd, const uint8_t* d_messages,
                                const uint8_t* d_signatures, uint32_t n, int32_t hash_kind, uint8_t* d_out_status);
/* Batch of PrivateKey::to_pub + PrivateKey::sign (mod.rs:206-237): per key 32 B secret scalar, 32 B randomness, 32 B message
 * -> compressed public key (x, is_odd), signature R.x || R.y || s.  out_status[i]: 1 = written; 2 = the reference returns
 * Err("Invalid repr") because s = (r + h a) mod ORDER does not fit the field (ORDER > r, mod.rs:222-233). */
int32_t og_bjj_sign_batch(og_ctx* ctx, const uint8_t* secret_keys, const uint8_t* randomness, const uint8_t* messages,
                          uint32_t n, int32_t hash_kind, uint8_t* out_pk_x, uint8_t* out_pk_is_odd,
                          uint8_t* out_signatures, uint8_t* out_status);
int32_t og_bjj_sign_batch_dev(og_ctx* ctx, const uint8_t* d_secret_keys, const uint8_t* d_randomness, const uint8_t* d_messages,
                              uint32_t n, int32_t hash_kind, uint8_t* d_out_pk_x, uint8_t* d_out_pk_is_odd,
                              uint8_t* d_out_signatures, uint8_t* d_out_status);

/* ---- Encrypted note delivery (DESIGN.md section 3, "Encrypted notes"; spec oracle/notes.py) ---------------------------
 * A view key v is a canonical Fr element with v mod l != 0 (l = the order of BASE); its public key (the address) is the
 * compressed point v BASE: x (32 B) and the parity of y (1 byte), exactly PrivateKey::to_pub.  A non-canonical view key
 * fails the call with OG_E_ENCODING, a key that is zero mod l with OG_E_INVALID.
 * A record is 160 B: E.x with the parity of E.y in bit 255, then c_0..c_3 (32 B little-endian words). */
int32_t og_note_public_keys(og_ctx* ctx, const uint8_t* view_keys, uint32_t n, uint8_t* out_pk_x, uint8_t* out_pk_is_odd);
/* One note per recipient key: nullifier, secret, token (32 B each), amount (u64), ephemeral scalar e (32 B) -> record,
 * commitment MultiMiMC7([nullifier, secret, token, amount], 0) (the transfer statement's output commitment) and
 * out_status[i]: 1 = written; 2 = the key does not decompress or 8 V = O; 3 = e = 0 mod l.  Refused notes get an all-zero
 * record and commitment.  Records and commitments must be 4-byte aligned in the _dev variant. */
int32_t og_note_encrypt(og_ctx* ctx, const uint8_t* pk_x, const uint8_t* pk_is_odd, const uint8_t* nullifiers, const uint8_t* secrets,
                        const uint8_t* tokens, const uint64_t* amounts, const uint8_t* ephemerals, uint64_t n,
                        uint8_t* out_records, uint8_t* out_commitments, uint8_t* out_status);
int32_t og_note_encrypt_dev(og_ctx* ctx, const uint8_t* d_pk_x, const uint8_t* d_pk_is_odd, const uint8_t* d_nullifiers, const uint8_t* d_secrets,
                            const uint8_t* d_tokens, const uint64_t* d_amounts, const uint8_t* d_ephemerals, uint64_t n,
                            uint8_t* d_out_records, uint8_t* d_out_commitments, uint8_t* d_out_status);
/* Trial-decrypt n records (with their commitments, 32 B each: the transfer proofs' out_commitment inputs) under n_keys
 * view keys (at most 65535).  out_owner[i]: the lowest index of a key that owns record i, 0xFFFFFFFF if none does,
 * 0xFFFFFFFE if the record is malformed (E.x >= r or bit 254 set, a c_i or the commitment >= r, E does not decompress,
 * 8 E = O).  out_plaintexts: 128 B per record, nullifier || secret || token || amount as field elements, zero unless owned.
 * view_keys is host memory in both variants (checked, then staged); the _dev variant's other buffers are device memory,
 * 4-byte aligned. */
int32_t og_note_scan(og_ctx* ctx, const uint8_t* view_keys, uint32_t n_keys, const uint8_t* records, const uint8_t* commitments,
                     uint64_t n, uint32_t* out_owner, uint8_t* out_plaintexts);
int32_t og_note_scan_dev(og_ctx* ctx, const uint8_t* view_keys, uint32_t n_keys, const uint8_t* d_records, const uint8_t* d_commitments,
                         uint64_t n, uint32_t* d_out_owner, uint8_t* d_out_plaintexts);
/* Spend-key notes (the owned transfer statement's, below): the same 160-byte record of the four words (owner P, blinding,
 * token, amount), its commitment MultiMiMC7([P, blinding, token, amount], 4) and status as og_note_encrypt's. */
int32_t og_owned_note_encrypt(og_ctx* ctx, const uint8_t* pk_x, const uint8_t* pk_is_odd, const uint8_t* owners, const uint8_t* blindings,
                              const uint8_t* tokens, const uint64_t* amounts, const uint8_t* ephemerals, uint64_t n,
                              uint8_t* out_records, uint8_t* out_commitments, uint8_t* out_status);
int32_t og_owned_note_encrypt_dev(og_ctx* ctx, const uint8_t* d_pk_x, const uint8_t* d_pk_is_odd, const uint8_t* d_owners,
                                  const uint8_t* d_blindings, const uint8_t* d_tokens, const uint64_t* d_amounts, const uint8_t* d_ephemerals,
                                  uint64_t n, uint8_t* d_out_records, uint8_t* d_out_commitments, uint8_t* d_out_status);
/* og_note_scan for spend-key notes: key k is a view key v_k with the spend public key P_k (32 B, canonical, else
 * OG_E_ENCODING) of the same wallet, and owns a record only if the record decrypts under v_k to an amount below 2^64, its
 * first word is P_k, and the key-4 commitment of the four words matches.  A note sent to v_k but to another spend key is
 * not owned: the wallet could not spend it.  view_keys and spend_public_keys are host memory in both variants. */
int32_t og_owned_note_scan(og_ctx* ctx, const uint8_t* view_keys, const uint8_t* spend_public_keys, uint32_t n_keys, const uint8_t* records,
                           const uint8_t* commitments, uint64_t n, uint32_t* out_owner, uint8_t* out_plaintexts);
int32_t og_owned_note_scan_dev(og_ctx* ctx, const uint8_t* view_keys, const uint8_t* spend_public_keys, uint32_t n_keys,
                               const uint8_t* d_records, const uint8_t* d_commitments, uint64_t n, uint32_t* d_out_owner,
                               uint8_t* d_out_plaintexts);
/* Owned labeled notes (the owned labeled transfer statement's, below): the same 160-byte record of the four words (owner P,
 * blinding, token, amount + 2^64 label), the note's key-7 leaf as commitment and status as og_note_encrypt's; labels are
 * uint32, one per note. */
int32_t og_owned_labeled_note_encrypt(og_ctx* ctx, const uint8_t* pk_x, const uint8_t* pk_is_odd, const uint8_t* owners,
                                      const uint8_t* blindings, const uint8_t* tokens, const uint64_t* amounts, const uint32_t* labels,
                                      const uint8_t* ephemerals, uint64_t n, uint8_t* out_records, uint8_t* out_commitments,
                                      uint8_t* out_status);
int32_t og_owned_labeled_note_encrypt_dev(og_ctx* ctx, const uint8_t* d_pk_x, const uint8_t* d_pk_is_odd, const uint8_t* d_owners,
                                          const uint8_t* d_blindings, const uint8_t* d_tokens, const uint64_t* d_amounts,
                                          const uint32_t* d_labels, const uint8_t* d_ephemerals, uint64_t n, uint8_t* d_out_records,
                                          uint8_t* d_out_commitments, uint8_t* d_out_status);
/* og_owned_note_scan for owned labeled notes: key k owns a record only if the record decrypts under v_k, word 3 is below
 * 2^96, the first word is P_k, and the key-7 leaf of (MultiMiMC7([m0, m1], 6), m2, word 3 mod 2^64, word 3 >> 64) matches.
 * A plaintext is the four words, word 3 = amount + 2^64 label. */
int32_t og_owned_labeled_note_scan(og_ctx* ctx, const uint8_t* view_keys, const uint8_t* spend_public_keys, uint32_t n_keys,
                                   const uint8_t* records, const uint8_t* commitments, uint64_t n, uint32_t* out_owner,
                                   uint8_t* out_plaintexts);
int32_t og_owned_labeled_note_scan_dev(og_ctx* ctx, const uint8_t* view_keys, const uint8_t* spend_public_keys, uint32_t n_keys,
                                       const uint8_t* d_records, const uint8_t* d_commitments, uint64_t n, uint32_t* d_out_owner,
                                       uint8_t* d_out_plaintexts);

/* ---- MSM (BASELINE configs 3 and 5) ----------------------------------------------------------- */
int32_t og_msm_g1(og_ctx* ctx, const uint8_t* points, const uint8_t* scalars, uint64_t n, uint8_t* out64);
int32_t og_msm_g2(og_ctx* ctx, const uint8_t* points, const uint8_t* scalars, uint64_t n, uint8_t* out128);
int32_t og_msm_g1_dev(og_ctx* ctx, const uint8_t* d_points, const uint8_t* d_scalars, uint64_t n, uint8_t* d_out64);
int32_t og_msm_g2_dev(og_ctx* ctx, const uint8_t* d_points, const uint8_t* d_scalars, uint64_t n, uint8_t* d_out128);
/* out_points[i] = scalars[i] * G for the standard generators (fixed-base windows on the GPU) */
int32_t og_g1_generator_mul(og_ctx* ctx, const uint8_t* scalars, uint64_t n, uint8_t* out_points64);
int32_t og_g2_generator_mul(og_ctx* ctx, const uint8_t* scalars, uint64_t n, uint8_t* out_points128);
int32_t og_g1_generator_mul_dev(og_ctx* ctx, const uint8_t* d_scalars, uint64_t n, uint8_t* d_out_points64);
int32_t og_g2_generator_mul_dev(og_ctx* ctx, const uint8_t* d_scalars, uint64_t n, uint8_t* d_out_points128);
/* plain sums of affine points: the local step after the multi-GPU all-gather of partial MSMs */
int32_t og_g1_sum(og_ctx* ctx, const uint8_t* points, uint64_t n, uint8_t* out64);
int32_t og_g2_sum(og_ctx* ctx, const uint8_t* points, uint64_t n, uint8_t* out128);
int32_t og_g1_sum_dev(og_ctx* ctx, const uint8_t* d_points, uint64_t n, uint8_t* d_out64);
int32_t og_g2_sum_dev(og_ctx* ctx, const uint8_t* d_points, uint64_t n, uint8_t* d_out128);

/* ---- NTT over Fr -------------------------------------------------------------------------------- */
/* `batch` independent transforms of 2^log_n elements, contiguous, natural order in and out.
 * omega = 7^((r-1)/2^log_n); coset = 1 evaluates on / interpolates from g*omega^k, g = omega_{2n}. */
int32_t og_ntt(og_ctx* ctx, uint8_t* data, uint32_t log_n, uint32_t batch, int32_t inverse, int32_t coset);
int32_t og_ntt_dev(og_ctx* ctx, uint8_t* d_data, uint32_t log_n, uint32_t batch, int32_t inverse, int32_t coset);

/* ---- the withdraw statement (DESIGN.md section 3) ---------------------------------------------- */
int32_t og_withdraw_r1cs_info(uint32_t depth, uint32_t* n_constraints, uint32_t* n_vars,
                              uint32_t* n_pub, uint32_t* log_m);
/* CSR of matrix `which` (0 = A, 1 = B, 2 = C); pass NULL arrays to query nnz only */
int32_t og_withdraw_r1cs_export(uint32_t depth, int32_t which, uint32_t* row_ptr, uint32_t* col_idx,
                                uint8_t* coeffs, uint64_t* nnz);
/* full assignments (batch * n_vars * 32 B) computed on the GPU */
int32_t og_withdraw_witness(og_ctx* ctx, uint32_t depth, const uint8_t* nullifiers, const uint8_t* secrets,
                            const uint8_t* recipients, const uint8_t* siblings, const uint32_t* path_bits,
                            uint32_t batch, uint8_t* witnesses);

/* ---- the deposit statement (DESIGN.md section 3): commitment = MultiMiMC7([nullifier, secret], 0) -- */
/* public inputs (commitment, depositor); 735 variables, 731 constraints, domain 2^10 */
int32_t og_deposit_r1cs_info(uint32_t* n_constraints, uint32_t* n_vars, uint32_t* n_pub, uint32_t* log_m);
/* CSR of matrix `which` (0 = A, 1 = B, 2 = C); pass NULL arrays to query nnz only */
int32_t og_deposit_r1cs_export(int32_t which, uint32_t* row_ptr, uint32_t* col_idx, uint8_t* coeffs, uint64_t* nnz);
/* full assignments (batch * n_vars * 32 B) computed on the GPU */
int32_t og_deposit_witness(og_ctx* ctx, const uint8_t* nullifiers, const uint8_t* secrets, const uint8_t* depositors,
                           uint32_t batch, uint8_t* witnesses);

/* ---- the transfer statement (DESIGN.md section 3): two value notes in, two out, a public amount --------------- */
/* note = (nullifier, secret, token, amount < 2^64), commitment = MultiMiMC7([nullifier, secret, token, amount], 0),
 * nullifier hash = MultiMiMC7([nullifier], 1).  Public inputs (root, public_amount, token, recipient, nullifier_hash[2],
 * out_commitment[2]); public_amount = out amounts - in amounts (mod r).  depth 1..32; at depth 32: 53 683 variables,
 * 53 609 constraints, domain 2^16. */
int32_t og_transfer_r1cs_info(uint32_t depth, uint32_t* n_constraints, uint32_t* n_vars, uint32_t* n_pub, uint32_t* log_m);
/* CSR of matrix `which` (0 = A, 1 = B, 2 = C); pass NULL arrays to query nnz only */
int32_t og_transfer_r1cs_export(uint32_t depth, int32_t which, uint32_t* row_ptr, uint32_t* col_idx, uint8_t* coeffs,
                                uint64_t* nnz);
/* full assignments (batch * n_vars * 32 B) computed on the GPU.  Per proof: roots / tokens / recipients 32 B each;
 * in_* and out_* hold note 0 then note 1 (nullifiers and secrets 2 * 32 B, amounts 2 * uint64); in_siblings holds
 * 2 * depth elements (input 0's path, then input 1's) and in_path_bits 2 words.  root is the caller's: an input of nonzero
 * amount that does not reach it, or two inputs with one nullifier, give a witness that does not satisfy the R1CS. */
int32_t og_transfer_witness(og_ctx* ctx, uint32_t depth, const uint8_t* roots, const uint8_t* tokens, const uint8_t* recipients,
                            const uint8_t* in_nullifiers, const uint8_t* in_secrets, const uint64_t* in_amounts,
                            const uint8_t* in_siblings, const uint32_t* in_path_bits,
                            const uint8_t* out_nullifiers, const uint8_t* out_secrets, const uint64_t* out_amounts,
                            uint32_t batch, uint8_t* witnesses);

/* ---- the association-set withdraw statement (DESIGN.md section 3): a note in the pool and in an approved subset ---- */
/* Public inputs (root, nullifier_hash, recipient, association_root); the first three are the withdraw statement's.  The
 * note's commitment MultiMiMC7([nullifier, secret], 0) reaches root along the pool path and association_root along the
 * path in an association set provider's tree over a subset of the deposits; both trees have the same depth, 1..32.  At
 * depth 32: 47 949 variables, 47 881 constraints, domain 2^16. */
int32_t og_association_r1cs_info(uint32_t depth, uint32_t* n_constraints, uint32_t* n_vars, uint32_t* n_pub, uint32_t* log_m);
/* CSR of matrix `which` (0 = A, 1 = B, 2 = C); pass NULL arrays to query nnz only */
int32_t og_association_r1cs_export(uint32_t depth, int32_t which, uint32_t* row_ptr, uint32_t* col_idx, uint8_t* coeffs,
                                   uint64_t* nnz);
/* full assignments (batch * n_vars * 32 B) computed on the GPU.  Per proof: nullifier, secret, recipient 32 B each; siblings
 * and assoc_siblings depth * 32 B each (leaf level first); path_bits and assoc_path_bits one word each (bit l set when the
 * level-l node is a right child).  Both roots are derived from the paths: a note that is not a leaf of a tree gives a root
 * that no one published. */
int32_t og_association_witness(og_ctx* ctx, uint32_t depth, const uint8_t* nullifiers, const uint8_t* secrets,
                               const uint8_t* recipients, const uint8_t* siblings, const uint32_t* path_bits,
                               const uint8_t* assoc_siblings, const uint32_t* assoc_path_bits, uint32_t batch, uint8_t* witnesses);

/* ---- the exclusion withdraw statement (DESIGN.md section 3): a note in the pool and not on a published blocklist ---- */
/* Public inputs (root, nullifier_hash, recipient, exclusion_root); the first three are the withdraw statement's.  A
 * provider's blocklist names pool leaf indices i_1 < ... < i_n; its tree (same depth as the pool's, 1..32) has leaf
 * j = MultiMiMC7([k_j, k_{j+1}], 0) over the keys k_0 = 0, k_j = i_j + 1, k_{n+1} = 2^32 + 1.  The note's commitment reaches
 * root along the pool path, its index i (the path bits) satisfies excl_low < i + 1 < excl_next (33-bit range checks), and the
 * leaf of (excl_low, excl_next) reaches exclusion_root along the exclusion path.  At depth 32: 48 812 variables,
 * 48 746 constraints, domain 2^16. */
int32_t og_exclusion_r1cs_info(uint32_t depth, uint32_t* n_constraints, uint32_t* n_vars, uint32_t* n_pub, uint32_t* log_m);
/* CSR of matrix `which` (0 = A, 1 = B, 2 = C); pass NULL arrays to query nnz only */
int32_t og_exclusion_r1cs_export(uint32_t depth, int32_t which, uint32_t* row_ptr, uint32_t* col_idx, uint8_t* coeffs,
                                 uint64_t* nnz);
/* full assignments (batch * n_vars * 32 B) computed on the GPU.  Per proof: nullifier, secret, recipient 32 B each; siblings
 * and excl_siblings depth * 32 B each (leaf level first); path_bits and excl_path_bits one word each (bit l set when the
 * level-l node is a right child; only the low depth bits count); excl_low and excl_next one uint64 each.  Both roots are
 * derived from the paths; a flagged note, a leaf that does not bracket the note, or a key of 2^33 or more gives a witness
 * that does not satisfy the R1CS. */
int32_t og_exclusion_witness(og_ctx* ctx, uint32_t depth, const uint8_t* nullifiers, const uint8_t* secrets,
                             const uint8_t* recipients, const uint8_t* siblings, const uint32_t* path_bits,
                             const uint64_t* excl_low, const uint64_t* excl_next, const uint8_t* excl_siblings,
                             const uint32_t* excl_path_bits, uint32_t batch, uint8_t* witnesses);

/* ---- labeled notes and the labeled withdraw statement (DESIGN.md section 3): partial withdrawals with change, checked
 * against a deposit blocklist ---- */
/* A labeled note is (nullifier, secret, token, amount < 2^64, label < 2^32); precommitment = MultiMiMC7([nullifier, secret], 2),
 * leaf = MultiMiMC7([precommitment, token, amount, label], 2).  The label is the pool leaf index at which the node appended
 * the deposit.  Wallet: precommitments of n notes (32 B each in and out). */
int32_t og_labeled_precommitments(og_ctx* ctx, const uint8_t* nullifiers, const uint8_t* secrets, uint64_t n, uint8_t* out);
/* Node: leaves of n deposits from precommitments and tokens (32 B each), amounts (uint64) and labels (uint32). */
int32_t og_labeled_leaves(og_ctx* ctx, const uint8_t* precommitments, const uint8_t* tokens, const uint64_t* amounts,
                          const uint32_t* labels, uint64_t n, uint8_t* out);
/* Public inputs (root, nullifier_hash, recipient, exclusion_root, token, withdrawn, change_commitment).  The note's leaf
 * reaches root along the pool path; amount, withdrawn and change = amount - withdrawn are range-checked to 64 bits and the
 * label to 32; change_commitment is the leaf of the change note (change_nullifier, change_secret, token, change, label);
 * x = label + 1 satisfies excl_low < x < excl_next (33-bit range checks) and the blocklist leaf of (excl_low, excl_next)
 * reaches exclusion_root (the exclusion statement's tree, same depth as the pool's, 1..32).  At depth 32: 52 685 variables,
 * 52 617 constraints, domain 2^16. */
int32_t og_labeled_r1cs_info(uint32_t depth, uint32_t* n_constraints, uint32_t* n_vars, uint32_t* n_pub, uint32_t* log_m);
/* CSR of matrix `which` (0 = A, 1 = B, 2 = C); pass NULL arrays to query nnz only */
int32_t og_labeled_r1cs_export(uint32_t depth, int32_t which, uint32_t* row_ptr, uint32_t* col_idx, uint8_t* coeffs,
                               uint64_t* nnz);
/* full assignments (batch * n_vars * 32 B) computed on the GPU.  Per proof: token, recipient 32 B each; withdrawn (uint64);
 * nullifier, secret 32 B each; amount (uint64); label (uint32); siblings depth * 32 B and path_bits one word (the note's
 * pool path); change_nullifier, change_secret 32 B each; excl_low, excl_next (uint64); excl_siblings depth * 32 B and
 * excl_path_bits one word (the blocklist path).  Path words: bit l set when the level-l node is a right child, only the low
 * depth bits count.  Both roots, the nullifier hash and change_commitment are derived; an overdraw, a flagged label or a
 * blocklist leaf that does not bracket it gives a witness that does not satisfy the R1CS. */
int32_t og_labeled_witness(og_ctx* ctx, uint32_t depth, const uint8_t* tokens, const uint8_t* recipients, const uint64_t* withdrawn,
                           const uint8_t* nullifiers, const uint8_t* secrets, const uint64_t* amounts, const uint32_t* labels,
                           const uint8_t* siblings, const uint32_t* path_bits, const uint8_t* change_nullifiers,
                           const uint8_t* change_secrets, const uint64_t* excl_low, const uint64_t* excl_next,
                           const uint8_t* excl_siblings, const uint32_t* excl_path_bits, uint32_t batch, uint8_t* witnesses);

/* ---- the labeled association withdraw statement (DESIGN.md section 3): partial withdrawals of labeled notes whose deposit
 * is on a provider's approved list ---- */
/* Public inputs (root, nullifier_hash, recipient, association_root, token, withdrawn, change_commitment).  The labeled
 * statement's note part (leaf under root, 64-bit ranges on amount, withdrawn and change, 32-bit range on the label, the
 * change note's commitment under the same label); then assoc_leaf = label + 1 reaches association_root in the provider's
 * tree of approved labels (leaf L + 1 per approved label L, every other leaf 0; same depth as the pool's, 1..32).  At depth
 * 32: 51 823 variables, 51 753 constraints, domain 2^16. */
int32_t og_labeled_association_r1cs_info(uint32_t depth, uint32_t* n_constraints, uint32_t* n_vars, uint32_t* n_pub, uint32_t* log_m);
/* CSR of matrix `which` (0 = A, 1 = B, 2 = C); pass NULL arrays to query nnz only */
int32_t og_labeled_association_r1cs_export(uint32_t depth, int32_t which, uint32_t* row_ptr, uint32_t* col_idx, uint8_t* coeffs,
                                           uint64_t* nnz);
/* full assignments (batch * n_vars * 32 B) computed on the GPU.  Per proof: token, recipient 32 B each; withdrawn (uint64);
 * nullifier, secret 32 B each; amount (uint64); label (uint32); siblings depth * 32 B and path_bits one word (the note's
 * pool path); change_nullifier, change_secret 32 B each; assoc_siblings depth * 32 B and assoc_path_bits one word (the path
 * of the label's leaf in the approved-label tree).  Path words: bit l set when the level-l node is a right child, only the
 * low depth bits count.  Both roots, the nullifier hash, assoc_leaf and change_commitment are derived; an overdraw or an
 * unapproved label gives a witness that does not satisfy the R1CS. */
int32_t og_labeled_association_witness(og_ctx* ctx, uint32_t depth, const uint8_t* tokens, const uint8_t* recipients,
                                       const uint64_t* withdrawn, const uint8_t* nullifiers, const uint8_t* secrets,
                                       const uint64_t* amounts, const uint32_t* labels, const uint8_t* siblings, const uint32_t* path_bits,
                                       const uint8_t* change_nullifiers, const uint8_t* change_secrets, const uint8_t* assoc_siblings,
                                       const uint32_t* assoc_path_bits, uint32_t batch, uint8_t* witnesses);

/* ---- spend-key notes and the owned transfer statement (DESIGN.md section 3): transfers whose outputs only the recipient's
 * spending key can spend ---- */
/* A spending key s is a canonical Fr element; its spend public key P = MultiMiMC7([s], 3).  A note is (P, blinding, token,
 * amount < 2^64) with commitment MultiMiMC7([P, blinding, token, amount], 4); spending it at leaf index i publishes the
 * nullifier MultiMiMC7([s, commitment, i], 5).  n items each, 32 B field elements in and out; indices uint32. */
int32_t og_owned_public_keys(og_ctx* ctx, const uint8_t* spend_keys, uint64_t n, uint8_t* out);
int32_t og_owned_commitments(og_ctx* ctx, const uint8_t* owners, const uint8_t* blindings, const uint8_t* tokens, const uint64_t* amounts,
                             uint64_t n, uint8_t* out);
int32_t og_owned_nullifiers(og_ctx* ctx, const uint8_t* spend_keys, const uint8_t* commitments, const uint32_t* indices, uint64_t n,
                            uint8_t* out);
/* The transfer statement's public inputs (root, public_amount, token, recipient, nullifier[2], out_commitment[2]), with
 * spend-key notes: each input proves knowledge of s for its note's owner, and nullifier[i] is its key-5 nullifier.  depth
 * 1..32; at depth 32: 55 867 variables, 55 793 constraints, domain 2^16. */
int32_t og_owned_transfer_r1cs_info(uint32_t depth, uint32_t* n_constraints, uint32_t* n_vars, uint32_t* n_pub, uint32_t* log_m);
/* CSR of matrix `which` (0 = A, 1 = B, 2 = C); pass NULL arrays to query nnz only */
int32_t og_owned_transfer_r1cs_export(uint32_t depth, int32_t which, uint32_t* row_ptr, uint32_t* col_idx, uint8_t* coeffs,
                                      uint64_t* nnz);
/* full assignments (batch * n_vars * 32 B) computed on the GPU.  Inputs as og_transfer_witness's with in_spend_keys and
 * in_blindings in place of in_nullifiers and in_secrets, out_owners (spend public keys) and out_blindings in place of
 * out_nullifiers and out_secrets.  root is the caller's: a wrong spend key, an input of nonzero amount that does not reach
 * root, or two inputs with one nullifier give a witness that does not satisfy the R1CS. */
int32_t og_owned_transfer_witness(og_ctx* ctx, uint32_t depth, const uint8_t* roots, const uint8_t* tokens, const uint8_t* recipients,
                                  const uint8_t* in_spend_keys, const uint8_t* in_blindings, const uint64_t* in_amounts,
                                  const uint8_t* in_siblings, const uint32_t* in_path_bits,
                                  const uint8_t* out_owners, const uint8_t* out_blindings, const uint64_t* out_amounts,
                                  uint32_t batch, uint8_t* witnesses);

/* ---- owned labeled notes and the owned labeled transfer statement (DESIGN.md section 3): private transfers of spend-key
 * notes that carry their deposit's label, checked against a provider's approved list ---- */
/* An owned labeled note is (P, blinding, token, amount < 2^64, label < 2^32): precommitment MultiMiMC7([P, blinding], 6),
 * leaf MultiMiMC7([precommitment, token, amount, label], 7); its nullifier is og_owned_nullifiers' of (s, leaf, index).
 * n items each, 32 B field elements in and out; amounts uint64, labels uint32. */
int32_t og_owned_labeled_precommitments(og_ctx* ctx, const uint8_t* owners, const uint8_t* blindings, uint64_t n, uint8_t* out);
int32_t og_owned_labeled_leaves(og_ctx* ctx, const uint8_t* precommitments, const uint8_t* tokens, const uint64_t* amounts,
                                const uint32_t* labels, uint64_t n, uint8_t* out);
/* Public inputs (root, association_root, token, withdrawn, recipient, nullifier[2], out_commitment[2]): two owned labeled
 * notes of one label in, two out under the same label, withdrawn (< 2^64) paid to recipient, in0 + in1 = out0 + out1 +
 * withdrawn, and label + 1 a leaf of the approved-label tree under association_root.  depth 1..32; at depth 32: 82 306
 * variables, 82 201 constraints, domain 2^17. */
int32_t og_owned_labeled_transfer_r1cs_info(uint32_t depth, uint32_t* n_constraints, uint32_t* n_vars, uint32_t* n_pub, uint32_t* log_m);
/* CSR of matrix `which` (0 = A, 1 = B, 2 = C); pass NULL arrays to query nnz only */
int32_t og_owned_labeled_transfer_r1cs_export(uint32_t depth, int32_t which, uint32_t* row_ptr, uint32_t* col_idx, uint8_t* coeffs,
                                              uint64_t* nnz);
/* full assignments (batch * n_vars * 32 B) computed on the GPU.  Per proof: root, token, recipient (32 B each), withdrawn
 * (uint64), label (uint32), in_spend_keys, in_blindings (2 x 32 B), in_amounts (2 x uint64), in_siblings (2 x depth x 32 B),
 * in_path_bits (2 x uint32), out_owners, out_blindings (2 x 32 B), out_amounts (2 x uint64), assoc_siblings (depth x 32 B),
 * assoc_path_bits (uint32).  root is the caller's and association_root is derived: a wrong spend key, an input of nonzero
 * amount that does not reach root under this label, an unapproved label, an overdraw or two inputs with one nullifier give
 * a witness that does not satisfy the R1CS. */
int32_t og_owned_labeled_transfer_witness(og_ctx* ctx, uint32_t depth, const uint8_t* roots, const uint8_t* tokens, const uint8_t* recipients,
                                          const uint64_t* withdrawn, const uint32_t* labels, const uint8_t* in_spend_keys,
                                          const uint8_t* in_blindings, const uint64_t* in_amounts, const uint8_t* in_siblings,
                                          const uint32_t* in_path_bits, const uint8_t* out_owners, const uint8_t* out_blindings,
                                          const uint64_t* out_amounts, const uint8_t* assoc_siblings, const uint32_t* assoc_path_bits,
                                          uint32_t batch, uint8_t* witnesses);

/* ---- the ragequit statement (DESIGN.md section 3): the public exit of an owned labeled note, with no provider approval ---- */
/* Public inputs (root, token, amount, label, recipient, nullifier): one owned labeled note (P = MultiMiMC7([s], 3), blinding,
 * token, amount, label) whose leaf reaches root, spent whole and paid to recipient; nullifier is og_owned_nullifiers' of
 * (s, leaf, index), the one an owned labeled transfer of the note would publish.  depth 1..32; at depth 32: 27 076
 * variables, 27 037 constraints, domain 2^15. */
int32_t og_ragequit_r1cs_info(uint32_t depth, uint32_t* n_constraints, uint32_t* n_vars, uint32_t* n_pub, uint32_t* log_m);
/* CSR of matrix `which` (0 = A, 1 = B, 2 = C); pass NULL arrays to query nnz only */
int32_t og_ragequit_r1cs_export(uint32_t depth, int32_t which, uint32_t* row_ptr, uint32_t* col_idx, uint8_t* coeffs, uint64_t* nnz);
/* full assignments (batch * n_vars * 32 B) computed on the GPU.  Per proof: root, token, recipient (32 B each), amount
 * (uint64), label (uint32), spend_key, blinding (32 B each), siblings (depth x 32 B), path_bits (uint32; only the low depth
 * bits count).  root is the caller's and the nullifier is derived: a wrong spend key, blinding, token, amount, label or path
 * gives a witness that does not satisfy the R1CS. */
int32_t og_ragequit_witness(og_ctx* ctx, uint32_t depth, const uint8_t* roots, const uint8_t* tokens, const uint8_t* recipients,
                            const uint64_t* amounts, const uint32_t* labels, const uint8_t* spend_keys, const uint8_t* blindings,
                            const uint8_t* siblings, const uint32_t* path_bits, uint32_t batch, uint8_t* witnesses);

/* ---- Groth16 ------------------------------------------------------------------------------------ */
/* Development ("toxic waste in the clear") setup for the withdraw statement, computed on the GPU.
 * toxic = tau || alpha || beta || gamma || delta (5 * 32 B).  Writes serialized pk / vk blobs;
 * call with pk_out == NULL to get the sizes. */
int32_t og_groth16_setup_withdraw(og_ctx* ctx, uint32_t depth, const uint8_t* toxic160,
                                  uint8_t* pk_out, uint64_t* pk_len, uint8_t* vk_out, uint64_t* vk_len);
/* The same setup for any R1CS: matrices A, B, C as CSR (row_ptr: n_constraints + 1 entries starting at 0, col < n_vars,
 * coefficients 32 B canonical), variable 0 = ONE, variables 1..n_pub the public inputs.  The key records depth 0.
 * OG_E_INVALID for a malformed CSR, n_constraints == 0, n_pub + 1 > n_vars, n_pub > 2^16, a domain above 2^24, or a
 * tau that puts tau or tau/g in the domain; OG_E_ENCODING for a coefficient >= r.  pk_out == NULL returns the sizes. */
int32_t og_groth16_setup(og_ctx* ctx, uint32_t n_constraints, uint32_t n_vars, uint32_t n_pub,
                         const uint32_t* a_row_ptr, const uint32_t* a_col, const uint8_t* a_coeffs,
                         const uint32_t* b_row_ptr, const uint32_t* b_col, const uint8_t* b_coeffs,
                         const uint32_t* c_row_ptr, const uint32_t* c_col, const uint8_t* c_coeffs,
                         const uint8_t* toxic160, uint8_t* pk_out, uint64_t* pk_len, uint8_t* vk_out, uint64_t* vk_len);
/* parse a pk blob, upload it and build the fixed-base window tables in HBM */
int32_t og_load_pk(og_ctx* ctx, const uint8_t* pk_bytes, uint64_t len, og_pk** out);
void og_free_pk(og_pk* pk);
int32_t og_pk_info(const og_pk* pk, uint32_t* n_vars, uint32_t* n_pub, uint32_t* log_m, uint32_t* depth);
/* window bits of the A (G1), B (G2) and C' (G1) MSMs the key proves with: chosen from the key's size when it was
 * loaded (OG_WINDOW_BITS / OG_C_A / OG_C_B / OG_C_C override) */
int32_t og_pk_window_bits(const og_pk* pk, uint32_t* c3);
/* how the prover runs `batch` proofs with this key: proofs per chunk, chunks in flight, and the scratch bytes of one lane.
 * Without OG_CHUNK the chunk is min(1024, 28 GiB / the scratch of one proof); OG_CHUNK / OG_LANES override. */
int32_t og_pk_prover_plan(const og_pk* pk, uint32_t batch, uint32_t* chunk, uint32_t* lanes, uint64_t* scratch_bytes_per_lane);

/* batch of proofs from full witnesses (batch * n_vars * 32 B); rs = batch * (r || s) */
int32_t og_groth16_prove(og_ctx* ctx, const og_pk* pk, const uint8_t* witnesses, uint32_t batch,
                         const uint8_t* rs, uint8_t* proofs);
/* batch of withdraw proofs from the secret inputs: witness generation (MiMC7 Merkle paths) runs on
 * the GPU too.  public_out (optional): batch * 3 * 32 B = root, nullifier_hash, recipient. */
int32_t og_groth16_prove_withdraw(og_ctx* ctx, const og_pk* pk, const uint8_t* nullifiers,
                                  const uint8_t* secrets, const uint8_t* recipients, const uint8_t* siblings,
                                  const uint32_t* path_bits, uint32_t batch, const uint8_t* rs,
                                  uint8_t* proofs, uint8_t* public_out);
/* same with every buffer already in HBM; no synchronisation */
int32_t og_groth16_prove_withdraw_dev(og_ctx* ctx, const og_pk* pk, const uint8_t* d_nullifiers,
                                      const uint8_t* d_secrets, const uint8_t* d_recipients,
                                      const uint8_t* d_siblings, const uint32_t* d_path_bits, uint32_t batch,
                                      const uint8_t* d_rs, uint8_t* d_proofs, uint8_t* d_public_out);
/* batch of deposit proofs from the secret inputs, witness generation on the GPU.  OG_E_INVALID unless the key has the
 * deposit statement's shape.  public_out (optional): batch * 2 * 32 B = commitment, depositor. */
int32_t og_groth16_prove_deposit(og_ctx* ctx, const og_pk* pk, const uint8_t* nullifiers, const uint8_t* secrets,
                                 const uint8_t* depositors, uint32_t batch, const uint8_t* rs, uint8_t* proofs,
                                 uint8_t* public_out);
/* same with every buffer already in HBM; no synchronisation */
int32_t og_groth16_prove_deposit_dev(og_ctx* ctx, const og_pk* pk, const uint8_t* d_nullifiers, const uint8_t* d_secrets,
                                     const uint8_t* d_depositors, uint32_t batch, const uint8_t* d_rs, uint8_t* d_proofs,
                                     uint8_t* d_public_out);
/* batch of transfer proofs from the notes, witness generation on the GPU; inputs as in og_transfer_witness.  OG_E_INVALID
 * unless the key has a transfer statement's shape (the depth is recognised from it).  public_out (optional):
 * batch * 8 * 32 B = root, public_amount, token, recipient, nullifier_hash[2], out_commitment[2]. */
int32_t og_groth16_prove_transfer(og_ctx* ctx, const og_pk* pk, const uint8_t* roots, const uint8_t* tokens,
                                  const uint8_t* recipients, const uint8_t* in_nullifiers, const uint8_t* in_secrets,
                                  const uint64_t* in_amounts, const uint8_t* in_siblings, const uint32_t* in_path_bits,
                                  const uint8_t* out_nullifiers, const uint8_t* out_secrets, const uint64_t* out_amounts,
                                  uint32_t batch, const uint8_t* rs, uint8_t* proofs, uint8_t* public_out);
/* same with every buffer already in HBM; no synchronisation */
int32_t og_groth16_prove_transfer_dev(og_ctx* ctx, const og_pk* pk, const uint8_t* d_roots, const uint8_t* d_tokens,
                                      const uint8_t* d_recipients, const uint8_t* d_in_nullifiers, const uint8_t* d_in_secrets,
                                      const uint64_t* d_in_amounts, const uint8_t* d_in_siblings, const uint32_t* d_in_path_bits,
                                      const uint8_t* d_out_nullifiers, const uint8_t* d_out_secrets, const uint64_t* d_out_amounts,
                                      uint32_t batch, const uint8_t* d_rs, uint8_t* d_proofs, uint8_t* d_public_out);
/* batch of association-set withdraw proofs, witness generation on the GPU; inputs as in og_association_witness.
 * OG_E_INVALID unless the key has an association statement's shape (the depth is recognised from it).  public_out
 * (optional): batch * 4 * 32 B = root, nullifier_hash, recipient, association_root. */
int32_t og_groth16_prove_association(og_ctx* ctx, const og_pk* pk, const uint8_t* nullifiers, const uint8_t* secrets,
                                     const uint8_t* recipients, const uint8_t* siblings, const uint32_t* path_bits,
                                     const uint8_t* assoc_siblings, const uint32_t* assoc_path_bits, uint32_t batch,
                                     const uint8_t* rs, uint8_t* proofs, uint8_t* public_out);
/* same with every buffer already in HBM; no synchronisation */
int32_t og_groth16_prove_association_dev(og_ctx* ctx, const og_pk* pk, const uint8_t* d_nullifiers, const uint8_t* d_secrets,
                                         const uint8_t* d_recipients, const uint8_t* d_siblings, const uint32_t* d_path_bits,
                                         const uint8_t* d_assoc_siblings, const uint32_t* d_assoc_path_bits, uint32_t batch,
                                         const uint8_t* d_rs, uint8_t* d_proofs, uint8_t* d_public_out);
/* batch of exclusion withdraw proofs, witness generation on the GPU; inputs as in og_exclusion_witness.  OG_E_INVALID
 * unless the key has an exclusion statement's shape (the depth is recognised from it).  public_out (optional):
 * batch * 4 * 32 B = root, nullifier_hash, recipient, exclusion_root. */
int32_t og_groth16_prove_exclusion(og_ctx* ctx, const og_pk* pk, const uint8_t* nullifiers, const uint8_t* secrets,
                                   const uint8_t* recipients, const uint8_t* siblings, const uint32_t* path_bits,
                                   const uint64_t* excl_low, const uint64_t* excl_next, const uint8_t* excl_siblings,
                                   const uint32_t* excl_path_bits, uint32_t batch, const uint8_t* rs, uint8_t* proofs,
                                   uint8_t* public_out);
/* same with every buffer already in HBM; no synchronisation */
int32_t og_groth16_prove_exclusion_dev(og_ctx* ctx, const og_pk* pk, const uint8_t* d_nullifiers, const uint8_t* d_secrets,
                                       const uint8_t* d_recipients, const uint8_t* d_siblings, const uint32_t* d_path_bits,
                                       const uint64_t* d_excl_low, const uint64_t* d_excl_next, const uint8_t* d_excl_siblings,
                                       const uint32_t* d_excl_path_bits, uint32_t batch, const uint8_t* d_rs, uint8_t* d_proofs,
                                       uint8_t* d_public_out);
/* batch of labeled withdraw proofs, witness generation on the GPU; inputs as in og_labeled_witness.  OG_E_INVALID unless
 * the key has a labeled statement's shape (the depth is recognised from it).  public_out (optional): batch * 7 * 32 B =
 * root, nullifier_hash, recipient, exclusion_root, token, withdrawn, change_commitment. */
int32_t og_groth16_prove_labeled(og_ctx* ctx, const og_pk* pk, const uint8_t* tokens, const uint8_t* recipients,
                                 const uint64_t* withdrawn, const uint8_t* nullifiers, const uint8_t* secrets, const uint64_t* amounts,
                                 const uint32_t* labels, const uint8_t* siblings, const uint32_t* path_bits,
                                 const uint8_t* change_nullifiers, const uint8_t* change_secrets, const uint64_t* excl_low,
                                 const uint64_t* excl_next, const uint8_t* excl_siblings, const uint32_t* excl_path_bits,
                                 uint32_t batch, const uint8_t* rs, uint8_t* proofs, uint8_t* public_out);
/* same with every buffer already in HBM; no synchronisation */
int32_t og_groth16_prove_labeled_dev(og_ctx* ctx, const og_pk* pk, const uint8_t* d_tokens, const uint8_t* d_recipients,
                                     const uint64_t* d_withdrawn, const uint8_t* d_nullifiers, const uint8_t* d_secrets,
                                     const uint64_t* d_amounts, const uint32_t* d_labels, const uint8_t* d_siblings,
                                     const uint32_t* d_path_bits, const uint8_t* d_change_nullifiers,
                                     const uint8_t* d_change_secrets, const uint64_t* d_excl_low, const uint64_t* d_excl_next,
                                     const uint8_t* d_excl_siblings, const uint32_t* d_excl_path_bits, uint32_t batch,
                                     const uint8_t* d_rs, uint8_t* d_proofs, uint8_t* d_public_out);
/* batch of labeled association withdraw proofs, witness generation on the GPU; inputs as in og_labeled_association_witness.
 * OG_E_INVALID unless the key has a labeled association statement's shape (the depth is recognised from it).  public_out
 * (optional): batch * 7 * 32 B = root, nullifier_hash, recipient, association_root, token, withdrawn, change_commitment. */
int32_t og_groth16_prove_labeled_association(og_ctx* ctx, const og_pk* pk, const uint8_t* tokens, const uint8_t* recipients,
                                             const uint64_t* withdrawn, const uint8_t* nullifiers, const uint8_t* secrets,
                                             const uint64_t* amounts, const uint32_t* labels, const uint8_t* siblings,
                                             const uint32_t* path_bits, const uint8_t* change_nullifiers, const uint8_t* change_secrets,
                                             const uint8_t* assoc_siblings, const uint32_t* assoc_path_bits, uint32_t batch,
                                             const uint8_t* rs, uint8_t* proofs, uint8_t* public_out);
/* same with every buffer already in HBM; no synchronisation */
int32_t og_groth16_prove_labeled_association_dev(og_ctx* ctx, const og_pk* pk, const uint8_t* d_tokens, const uint8_t* d_recipients,
                                                 const uint64_t* d_withdrawn, const uint8_t* d_nullifiers, const uint8_t* d_secrets,
                                                 const uint64_t* d_amounts, const uint32_t* d_labels, const uint8_t* d_siblings,
                                                 const uint32_t* d_path_bits, const uint8_t* d_change_nullifiers,
                                                 const uint8_t* d_change_secrets, const uint8_t* d_assoc_siblings,
                                                 const uint32_t* d_assoc_path_bits, uint32_t batch, const uint8_t* d_rs,
                                                 uint8_t* d_proofs, uint8_t* d_public_out);
/* batch of owned transfer proofs, witness generation on the GPU; inputs as in og_owned_transfer_witness.  OG_E_INVALID unless
 * the key has an owned transfer statement's shape (the depth is recognised from it).  public_out (optional): batch * 8 * 32 B
 * = root, public_amount, token, recipient, nullifier[2], out_commitment[2]. */
int32_t og_groth16_prove_owned_transfer(og_ctx* ctx, const og_pk* pk, const uint8_t* roots, const uint8_t* tokens, const uint8_t* recipients,
                                        const uint8_t* in_spend_keys, const uint8_t* in_blindings, const uint64_t* in_amounts,
                                        const uint8_t* in_siblings, const uint32_t* in_path_bits,
                                        const uint8_t* out_owners, const uint8_t* out_blindings, const uint64_t* out_amounts,
                                        uint32_t batch, const uint8_t* rs, uint8_t* proofs, uint8_t* public_out);
int32_t og_groth16_prove_owned_transfer_dev(og_ctx* ctx, const og_pk* pk, const uint8_t* d_roots, const uint8_t* d_tokens,
                                            const uint8_t* d_recipients, const uint8_t* d_in_spend_keys, const uint8_t* d_in_blindings,
                                            const uint64_t* d_in_amounts, const uint8_t* d_in_siblings, const uint32_t* d_in_path_bits,
                                            const uint8_t* d_out_owners, const uint8_t* d_out_blindings, const uint64_t* d_out_amounts,
                                            uint32_t batch, const uint8_t* d_rs, uint8_t* d_proofs, uint8_t* d_public_out);
/* batch of owned labeled transfer proofs, witness generation on the GPU; inputs as in og_owned_labeled_transfer_witness.
 * OG_E_INVALID unless the key has an owned labeled transfer statement's shape (the depth is recognised from it).
 * public_out (optional): batch * 9 * 32 B = root, association_root, token, withdrawn, recipient, nullifier[2],
 * out_commitment[2]. */
int32_t og_groth16_prove_owned_labeled_transfer(og_ctx* ctx, const og_pk* pk, const uint8_t* roots, const uint8_t* tokens,
                                                const uint8_t* recipients, const uint64_t* withdrawn, const uint32_t* labels,
                                                const uint8_t* in_spend_keys, const uint8_t* in_blindings, const uint64_t* in_amounts,
                                                const uint8_t* in_siblings, const uint32_t* in_path_bits, const uint8_t* out_owners,
                                                const uint8_t* out_blindings, const uint64_t* out_amounts, const uint8_t* assoc_siblings,
                                                const uint32_t* assoc_path_bits, uint32_t batch, const uint8_t* rs, uint8_t* proofs,
                                                uint8_t* public_out);
int32_t og_groth16_prove_owned_labeled_transfer_dev(og_ctx* ctx, const og_pk* pk, const uint8_t* d_roots, const uint8_t* d_tokens,
                                                    const uint8_t* d_recipients, const uint64_t* d_withdrawn, const uint32_t* d_labels,
                                                    const uint8_t* d_in_spend_keys, const uint8_t* d_in_blindings, const uint64_t* d_in_amounts,
                                                    const uint8_t* d_in_siblings, const uint32_t* d_in_path_bits, const uint8_t* d_out_owners,
                                                    const uint8_t* d_out_blindings, const uint64_t* d_out_amounts,
                                                    const uint8_t* d_assoc_siblings, const uint32_t* d_assoc_path_bits, uint32_t batch,
                                                    const uint8_t* d_rs, uint8_t* d_proofs, uint8_t* d_public_out);
/* batch of ragequit proofs, witness generation on the GPU; inputs as in og_ragequit_witness.  OG_E_INVALID unless the key
 * has a ragequit statement's shape (the depth is recognised from it).  public_out (optional): batch * 6 * 32 B = root,
 * token, amount, label, recipient, nullifier. */
int32_t og_groth16_prove_ragequit(og_ctx* ctx, const og_pk* pk, const uint8_t* roots, const uint8_t* tokens, const uint8_t* recipients,
                                  const uint64_t* amounts, const uint32_t* labels, const uint8_t* spend_keys, const uint8_t* blindings,
                                  const uint8_t* siblings, const uint32_t* path_bits, uint32_t batch, const uint8_t* rs, uint8_t* proofs,
                                  uint8_t* public_out);
int32_t og_groth16_prove_ragequit_dev(og_ctx* ctx, const og_pk* pk, const uint8_t* d_roots, const uint8_t* d_tokens, const uint8_t* d_recipients,
                                      const uint64_t* d_amounts, const uint32_t* d_labels, const uint8_t* d_spend_keys,
                                      const uint8_t* d_blindings, const uint8_t* d_siblings, const uint32_t* d_path_bits, uint32_t batch,
                                      const uint8_t* d_rs, uint8_t* d_proofs, uint8_t* d_public_out);
/* debug/parity probe: the H-query scalars d_j = (a*b - c)(g w^j) for one witness, 2^log_m * 32 B */
int32_t og_groth16_h_evals(og_ctx* ctx, const og_pk* pk, const uint8_t* witness, uint8_t* out);

/* host-side verifier (3 pairings + n_pub scalar multiplications): OG_OK or OG_E_VERIFY */
int32_t og_groth16_verify(const uint8_t* vk, uint64_t vk_len, const uint8_t* public_inputs,
                          uint32_t n_pub, const uint8_t* proof256);

/* ---- two-phase setup ceremony (DESIGN.md section 4b) ----------------------------------------------------------------
 * Phase 1: a powers-of-tau accumulator ("OGPT" v1, log_max in [1, 24], M = 2^log_max): [tau^i]_1 (i < 2M),
 * [alpha tau^i]_1, [beta tau^i]_1, [tau^i]_2 (i < M), [beta]_2.  og_ptau_new makes the initial one (all generators);
 * og_ptau_contribute applies secrets (t, a, b) and writes a record ("OGPR" v1) with Schnorr proofs of knowledge made with
 * the nonces (96 bytes each: three 32-byte scalars); og_ptau_verify checks one update against its record.
 * og_ptau_prepare / og_ptau_prepare_withdraw derive a circuit's key (gamma = delta = 1) from an accumulator whose
 * log_max is at least the circuit's log_m.  Phase 2: og_phase2_contribute multiplies delta by d (L and H by 1/d) and
 * writes a record ("OGDR" v1); og_phase2_verify checks it.  Verification returns OG_OK or OG_E_VERIFY.  Outputs follow
 * the NULL -> size convention; zero secrets or nonces, malformed blobs and m > M give OG_E_INVALID.  The library zeroes
 * its copies of the secrets before returning. */
int32_t og_ptau_new(og_ctx* ctx, uint32_t log_max, uint8_t* out, uint64_t* out_len);
int32_t og_ptau_contribute(og_ctx* ctx, const uint8_t* acc, uint64_t acc_len, const uint8_t* secrets96, const uint8_t* nonces96,
                           uint8_t* acc_out, uint64_t* acc_out_len, uint8_t* record_out, uint64_t* record_len);
int32_t og_ptau_verify(og_ctx* ctx, const uint8_t* prev, uint64_t prev_len, const uint8_t* next, uint64_t next_len,
                       const uint8_t* record, uint64_t record_len);
int32_t og_ptau_prepare(og_ctx* ctx, const uint8_t* acc, uint64_t acc_len, uint32_t n_constraints, uint32_t n_vars, uint32_t n_pub,
                        const uint32_t* a_row_ptr, const uint32_t* a_col, const uint8_t* a_coeffs,
                        const uint32_t* b_row_ptr, const uint32_t* b_col, const uint8_t* b_coeffs,
                        const uint32_t* c_row_ptr, const uint32_t* c_col, const uint8_t* c_coeffs,
                        uint8_t* pk_out, uint64_t* pk_len, uint8_t* vk_out, uint64_t* vk_len);
int32_t og_ptau_prepare_withdraw(og_ctx* ctx, const uint8_t* acc, uint64_t acc_len, uint32_t depth, uint8_t* pk_out, uint64_t* pk_len,
                                 uint8_t* vk_out, uint64_t* vk_len);
int32_t og_phase2_contribute(og_ctx* ctx, const uint8_t* pk, uint64_t pk_len, const uint8_t* vk, uint64_t vk_len, const uint8_t* delta32,
                             const uint8_t* nonce32, uint8_t* pk_out, uint64_t* pk_out_len, uint8_t* vk_out, uint64_t* vk_out_len,
                             uint8_t* record_out, uint64_t* record_len);
int32_t og_phase2_verify(og_ctx* ctx, const uint8_t* pk_prev, uint64_t pk_prev_len, const uint8_t* vk_prev, uint64_t vk_prev_len,
                         const uint8_t* pk_next, uint64_t pk_next_len, const uint8_t* vk_next, uint64_t vk_next_len,
                         const uint8_t* record, uint64_t record_len);
/* the ceremony's point kernels: out_i = s_i P_i (per_point) or s_0 P_i over G1 (g2 = 0) or G2 (g2 = 1), and the in-place
 * inverse NTT of 2^log_m points (omega = 7^((r-1)/m), as og_ntt) */
int32_t og_scale_points(og_ctx* ctx, int32_t g2, const uint8_t* points, const uint8_t* scalars, uint64_t n, int32_t per_point,
                        uint8_t* out);
int32_t og_intt_points(og_ctx* ctx, int32_t g2, uint8_t* points, uint32_t log_m);

/* ---- test/debug probes of the MSM engine (not for integrators) ----------------------------------------------------------
 * og_msm_bucket_sums runs the bucket stage of the G1 (g2 = 0) or G2 (g2 = 1) MSM -- bucket order, accumulation, heavy buckets,
 * reduction -- on bucket lists the caller gives.  counts: n_groups * nb list lengths (key = g * nb + b); entries: sum(counts)
 * words in key order, (point index << 1) | negate.  out_totals: n_groups affine points sum_b (b + 1) B_b; out_buckets (NULL
 * to skip): the n_groups * nb buckets after accumulation and heavy combine.  few_groups selects the one-shot MSM's reduction
 * (the tree-sum tail).  OG_E_INVALID, before anything is launched, unless nb is a power of two in [2, 2^15], n_groups is in
 * [1, 65535], n_groups * nb <= 2^26, every point index is below n_points, sum(counts) < 2^32,
 * sum(counts) <= n_entries_max < 2^30, and the heavy buckets' segments fit the engine's level scratch (the heavy-bucket cap and
 * segment length follow n_entries_max / (n_groups * nb); a plan over that scratch needs an average of 512 or more entries per key). */
int32_t og_msm_bucket_sums(og_ctx* ctx, int32_t g2, const uint8_t* points, uint32_t n_points, const uint32_t* counts,
                           const uint32_t* entries, uint32_t n_groups, uint32_t nb, uint64_t n_entries_max, int32_t few_groups,
                           uint8_t* out_totals, uint8_t* out_buckets);
/* Element-wise arithmetic of the MSM units on raw Montgomery limbs (no conversion, no range check), through the functions the bucket
 * kernels call (the same source and PTX; the compiler gives each kernel its own machine-code copy of them).  unit 0 (G1 unit, Fq, 32 B per operand): op 0 a * b, 1 a^2, 2 a - b, 3 a + a
 * (canonical forms), 8 lazy a * b, 9 lazy a^2 (the out-of-line squarer), 10 lazy a + b, 11 lazy a - b, 12 a reduced to [0, p),
 * 13 "a == 0 mod p" (1 or 0 in the first byte, the rest zero), 14 lazy a^2 + (2p - b)^2 with one reduction; ops 4-7 are invalid.
 * unit 1 (G2 unit, Fq2, 64 B): op 0 lazy a * b, 1 lazy a^2, 2 lazy a + b, 3 lazy a - b, 4 a reduced to [0, p), 5 a * b,
 * 6 a^2, 7 "a == 0 mod p" (1 or 0 in the first byte, the rest zero).  b is read for every op. */
int32_t og_field_probe_raw(og_ctx* ctx, int32_t unit, int32_t op, const uint8_t* a, const uint8_t* b, uint64_t n, uint8_t* out);

#ifdef __cplusplus
}
#endif
#endif
