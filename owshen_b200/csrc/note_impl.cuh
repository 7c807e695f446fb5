// owshen_b200/csrc/note_impl.cuh -- (included at the end of mimc.cu, after bjj_impl.cuh: it shares the MiMC7 round constants
// and the BabyJubJub fixed-base table) encrypted note delivery on sm_90a (DESIGN.md sections 3 and 5.6; spec: oracle/notes.py).
//
//   k_note_public_keys   one thread per view key: v BASE through the fixed-base table
//   k_note_encrypt       one thread per note
//   k_note_prepare       one thread per record: parse, decompress E, E' = 8 E and the malformed checks, once for all keys;
//                        writes E' (the only scratch) and seeds the owner word with NOT_OWNED or MALFORMED
//   k_note_scan          one thread per (record, key); blockIdx.y is the key, so a warp shares one scalar and the
//                        window digits never diverge.  An owner is recorded with atomicMin, so the
//                        lowest owning key index wins whatever the scheduling
//   k_note_finish        one thread per record: zero plaintext, or the note decrypted again under the winning key
// The encrypt, scan and finish kernels take the note kind: transfer notes (commitment key 0), spend-key notes (commitment key
// 4) and owned labeled notes (the key-7 leaf, word 3 = amount + 2^64 label); for the last two a record is owned by key k only
// if its m0 is the spend public key P_k as well.
#include "note_core.cuh"

namespace og {

struct NoteC {                                        // the round constants, as the `c(i)` of note_core.cuh
    __device__ __forceinline__ Fr operator()(int i) const { return mimc_c(i); }
};

__global__ void __launch_bounds__(64) k_note_public_keys(const Fr* __restrict__ base_tab, const uint8_t* __restrict__ keys, uint32_t n,
                                                         uint8_t* __restrict__ pk_x, uint8_t* __restrict__ pk_odd, int* flag) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Fr v = load_canonical<Fr>(keys + 32ull * i, flag), x, y;
    const BjjBase base{Fr::zero(), Fr::zero(), base_tab};
    bjj_to_pub(&x, &y, &base, &v);
    store_canonical(pk_x + 32ull * i, x);
    pk_odd[i] = fr_is_odd(y) ? 1 : 0;
}

// labels: one label per note for NOTE_OWNED_LABELED (word 3 = amount + 2^64 label), unread otherwise
template <NoteKind KIND>
__global__ void __launch_bounds__(64) k_note_encrypt(const Fr* __restrict__ base_tab, NoteEncryptInputs in, uint64_t n,
                                                     uint8_t* __restrict__ records, uint8_t* __restrict__ commitments,
                                                     uint8_t* __restrict__ status, int* flag, const uint32_t* __restrict__ labels) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint64_t amount = in.amounts[i];
    uint32_t a[8] = {(uint32_t)amount, (uint32_t)(amount >> 32), KIND == NOTE_OWNED_LABELED ? labels[i] : 0, 0, 0, 0, 0, 0};
    Fr m[4] = {load_canonical<Fr>(in.nullifiers + 32 * i, flag), load_canonical<Fr>(in.secrets + 32 * i, flag),
               load_canonical<Fr>(in.tokens + 32 * i, flag), Fr::from_canonical(a)};
    Fr pk_x = load_canonical<Fr>(in.pk_x + 32 * i, flag), e = load_canonical<Fr>(in.ephemerals + 32 * i, flag), cm;
    uint32_t w[NOTE_RECORD_WORDS];
    status[i] = note_encrypt_one<note_kind_key(KIND)>(pk_x, in.pk_odd[i] != 0, m, e, BjjBase{Fr::zero(), Fr::zero(), base_tab},
                                                      NoteC{}, w, &cm);
    uint32_t* out = reinterpret_cast<uint32_t*>(records + 160 * i);
#pragma unroll
    for (uint32_t k = 0; k < NOTE_RECORD_WORDS; k++) out[k] = w[k];
    store_canonical(commitments + 32 * i, cm);
}

__global__ void __launch_bounds__(128) k_note_prepare(const uint8_t* __restrict__ records, const uint8_t* __restrict__ commitments,
                                                      uint64_t n, Fr* __restrict__ prepared, uint32_t* __restrict__ owner) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Fr x, y;
    bool ok = note_prepare_one(reinterpret_cast<const uint32_t*>(records + 160 * i), reinterpret_cast<const uint32_t*>(commitments + 32 * i),
                               &x, &y);
    prepared[2 * i] = ok ? x : Fr::zero();
    prepared[2 * i + 1] = ok ? y : Fr::one();
    owner[i] = ok ? NOTE_NOT_OWNED : NOTE_MALFORMED;
}

template <NoteKind KIND>
__global__ void __launch_bounds__(64) k_note_scan(const uint32_t* __restrict__ keys, const uint32_t* __restrict__ spend_keys,
                                                  const uint8_t* __restrict__ records, const uint8_t* __restrict__ commitments,
                                                  const Fr* __restrict__ prepared, uint64_t n, uint32_t* owner) {
    const uint32_t key = blockIdx.y;
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || owner[i] == NOTE_MALFORMED) return;     // MALFORMED is written by k_note_prepare only, never by atomicMin
    uint32_t v[8];
#pragma unroll
    for (int k = 0; k < 8; k++) v[k] = keys[8 * key + k];
    Fr m[4];
    if (note_decrypt_one<true, note_kind_key(KIND)>(prepared[2 * i], prepared[2 * i + 1], v,
                                                    reinterpret_cast<const uint32_t*>(records + 160 * i),
                                                    reinterpret_cast<const uint32_t*>(commitments + 32 * i), NoteC{}, m) &&
        (KIND == NOTE_TRANSFER || m[0] == Fr::from_canonical(spend_keys + 8 * key)))
        atomicMin(owner + i, key);
}

template <NoteKind KIND>
__global__ void __launch_bounds__(64) k_note_finish(const uint32_t* __restrict__ keys, uint32_t n_keys, const uint8_t* __restrict__ records,
                                                    const uint8_t* __restrict__ commitments, const Fr* __restrict__ prepared, uint64_t n,
                                                    const uint32_t* __restrict__ owner, uint8_t* __restrict__ plaintexts) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t o = owner[i];
    Fr m[4] = {Fr::zero(), Fr::zero(), Fr::zero(), Fr::zero()};
    if (o < n_keys)
        note_decrypt_one<false, note_kind_key(KIND)>(prepared[2 * i], prepared[2 * i + 1], keys + 8ull * o,
                                                     reinterpret_cast<const uint32_t*>(records + 160 * i),
                                                     reinterpret_cast<const uint32_t*>(commitments + 32 * i), NoteC{}, m);
    for (int k = 0; k < 4; k++) store_canonical(plaintexts + 128 * i + 32 * k, m[k]);
}

// ---- host side ------------------------------------------------------------------------------------
// a view key must be canonical (OG_E_ENCODING) and nonzero mod l (OG_E_INVALID); v < r < 8 l, so the multiples to refuse are
// 0, l, ..., 7 l, with l = ORDER / 8
int32_t note_check_view_keys(og_ctx* ctx, const uint8_t* keys, uint32_t n) {
    uint32_t l[8];
    for (int i = 0; i < 8; i++) l[i] = (bjj_order_limb(i) >> 3) | (i < 7 ? bjj_order_limb(i + 1) << 29 : 0);
    for (uint32_t j = 0; j < n; j++) {
        uint32_t v[8];
        memcpy(v, keys + 32ull * j, 32);
        if (!Fr::canonical_lt_mod(v)) {
            snprintf(ctx->err, sizeof(ctx->err), "view key %u is not a canonical field element", j);
            return OG_E_ENCODING;
        }
        uint32_t kl[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        for (int k = 0; k < 8; k++) {
            if (memcmp(kl, v, 32) == 0) {
                snprintf(ctx->err, sizeof(ctx->err), "view key %u is zero mod the subgroup order l", j);
                return OG_E_INVALID;
            }
            uint64_t c = 0;
            for (int t = 0; t < 8; t++) { c += (uint64_t)kl[t] + l[t]; kl[t] = (uint32_t)c; c >>= 32; }
        }
    }
    return OG_OK;
}

int32_t note_public_keys_dev(og_ctx* ctx, const uint8_t* d_keys, uint32_t n, uint8_t* d_pk_x, uint8_t* d_pk_odd) {
    if (n == 0) return OG_OK;
    const Fr* tab;
    OG_TRY(bjj_table(ctx, &tab));
    OG_LAUNCH(ctx, k_note_public_keys, (n + 63) / 64, 64, 0, tab, d_keys, n, d_pk_x, d_pk_odd, ctx->d_flag);
    return OG_OK;
}

// the note kinds' og_profile names: the transfer-note kernels keep theirs, the other kinds' are k_owned_note_* and
// k_owned_labeled_note_*
struct NoteKernelNames { const char *encrypt, *scan, *finish; };
constexpr NoteKernelNames NOTE_KERNEL_NAMES[] = {
    {"k_note_encrypt", "k_note_scan", "k_note_finish"},
    {"k_owned_note_encrypt", "k_owned_note_scan", "k_owned_note_finish"},
    {"k_owned_labeled_note_encrypt", "k_owned_labeled_note_scan", "k_owned_labeled_note_finish"},
};

// f(std::integral_constant<NoteKind, kind>): the kernels' template argument from the kind a call names
template <class F>
static int32_t with_note_kind(NoteKind kind, F&& f) {
    switch (kind) {
    case NOTE_TRANSFER: return f(std::integral_constant<NoteKind, NOTE_TRANSFER>{});
    case NOTE_OWNED: return f(std::integral_constant<NoteKind, NOTE_OWNED>{});
    case NOTE_OWNED_LABELED: return f(std::integral_constant<NoteKind, NOTE_OWNED_LABELED>{});
    }
    return OG_E_INVALID;
}

int32_t note_encrypt_dev(og_ctx* ctx, const NoteEncryptInputs& in, uint64_t n, uint8_t* d_records, uint8_t* d_commitments, uint8_t* d_status,
                         NoteKind kind, const uint32_t* d_labels) {
    if (n == 0) return OG_OK;
    const Fr* tab;
    OG_TRY(bjj_table(ctx, &tab));
    return with_note_kind(kind, [&](auto k) -> int32_t {
        constexpr NoteKind KIND = decltype(k)::value;
        OG_LAUNCHN(ctx, NOTE_KERNEL_NAMES[KIND].encrypt, k_note_encrypt<KIND>, (unsigned)((n + 63) / 64), 64, 0, tab, in, n, d_records,
                   d_commitments, d_status, ctx->d_flag, d_labels);
        return OG_OK;
    });
}

// d_keys: n_keys checked view keys (canonical limbs) in device memory, and d_spend_keys their checked spend public keys for
// spend-key and owned labeled notes (unread for transfer notes); the prepared points go to a context slot.  The
// variable-base multiplier is the 4-bit window (DESIGN.md section 5.6).
int32_t note_scan_dev(og_ctx* ctx, const uint32_t* d_keys, uint32_t n_keys, const uint8_t* d_records, const uint8_t* d_commitments, uint64_t n,
                      uint32_t* d_owner, uint8_t* d_plaintexts, NoteKind kind, const uint32_t* d_spend_keys) {
    if (n == 0) return OG_OK;
    if (n_keys > 65535) { snprintf(ctx->err, sizeof(ctx->err), "at most 65535 view keys per scan"); return OG_E_INVALID; }
    OG_SLOT(ctx, prep, Fr, S_NOTE_PREP, sizeof(Fr) * 2 * n);
    const unsigned blocks = (unsigned)((n + 63) / 64);
    OG_LAUNCH(ctx, k_note_prepare, (unsigned)((n + 127) / 128), 128, 0, d_records, d_commitments, n, prep, d_owner);
    return with_note_kind(kind, [&](auto k) -> int32_t {
        constexpr NoteKind KIND = decltype(k)::value;
        if (n_keys)
            OG_LAUNCHN(ctx, NOTE_KERNEL_NAMES[KIND].scan, k_note_scan<KIND>, dim3(blocks, n_keys), 64, 0, d_keys, d_spend_keys, d_records,
                       d_commitments, prep, n, d_owner);
        OG_LAUNCHN(ctx, NOTE_KERNEL_NAMES[KIND].finish, k_note_finish<KIND>, blocks, 64, 0, d_keys, n_keys, d_records, d_commitments, prep, n,
                   d_owner, d_plaintexts);
        return OG_OK;
    });
}

}  // namespace og
