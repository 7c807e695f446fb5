// owshen_b200/csrc/note_core.cuh -- encrypted note delivery (DESIGN.md section 3, "Encrypted notes"; spec: oracle/notes.py),
// host+device so that tests run the exact code on a CPU (tests/harness/note_harness.cpp).
//
//   encrypt (sender)   V' = 8 V, E = e BASE, S = affine(e V'), k = MultiMiMC7([S.x, S.y]), c_i = m_i + MiMC7(i, k)
//   prepare (per record, once for all keys)   parse word 0, decompress E, E' = affine(8 E), range checks
//   decrypt (per record and key)   S = affine(v E'), m_i = c_i - MiMC7(i, k), owned iff amount < 2^64 and
//                                  MultiMiMC7(m) equals the commitment
// `c(i)` returns MiMC7 round constant i (Montgomery form), as in mimc_core.cuh.  Records are 40 little-endian 32-bit words:
// word 0 (8 limbs) is E.x with the parity of E.y in bit 255, words 1..4 are c_0..c_3.
#pragma once
#include "bjj_core.cuh"
#include "mimc_core.cuh"

namespace og {

constexpr uint32_t NOTE_RECORD_WORDS = 40;            // 160 bytes
constexpr uint32_t NOTE_NOT_OWNED = 0xFFFFFFFFu, NOTE_MALFORMED = 0xFFFFFFFEu;
enum : uint8_t { NOTE_ENC_OK = 1, NOTE_ENC_BAD_KEY = 2, NOTE_ENC_BAD_EPHEMERAL = 3 };

OG_HD bool bjj_is_identity(const Fr& x, const Fr& y) { return x.is_zero() && y == Fr::one(); }

// affine(8 P) for an affine point P: the three doublings that clear the cofactor
OG_HD void note_clear_cofactor(Fr* x, Fr* y, const Fr& px, const Fr& py) {
    const Fr A = bjj_a();
    BjjPoint p{px, py, Fr::one()};
    for (int i = 0; i < 3; i++) bjj_double(&p, &A);
    bjj_to_affine(x, y, &p);
}

// k = MultiMiMC7([S.x, S.y], 0) and the four pads MiMC7(i, k) = perm(i, k) + k
template <class CFn>
OG_HD void note_pads(Fr pad[4], const Fr& sx, const Fr& sy, CFn c) {
    Fr k = mimc7_hash2_lazy(sx, sy, c);
    for (uint32_t i = 0; i < 4; i++) pad[i] = mimc7_perm_lazy<false>(Fr::from_u32(i), k, c);
}

// KEY 7 names the owned labeled note (oracle/owned_labeled_circuit.py): its words are (owner, blinding, token, amount + 2^64
// label), word 3 may reach 2^96, and its commitment is the leaf MultiMiMC7([MultiMiMC7([owner, blinding], 6), token, amount,
// label], 7)
constexpr uint32_t NOTE_LABELED_KEY = 7;

template <class CFn>
OG_HD Fr note_labeled_leaf(const Fr m[4], CFn c) {
    const Fr k6 = Fr::from_u32(6), k7 = Fr::from_u32(NOTE_LABELED_KEY);
    Fr pre = k6 + m[0] + mimc7_perm_lazy<false>(m[0], k6, c);
    pre = pre + m[1] + mimc7_perm_lazy<false>(m[1], pre, c);
    uint32_t a[8], lo[8] = {0, 0, 0, 0, 0, 0, 0, 0}, hi[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    m[3].to_canonical(a);
    lo[0] = a[0]; lo[1] = a[1]; hi[0] = a[2];
    const Fr xs[3] = {m[2], Fr::from_canonical(lo), Fr::from_canonical(hi)};
    Fr r = k7 + pre + mimc7_perm_lazy<false>(pre, k7, c);
    for (int i = 0; i < 3; i++) r = r + xs[i] + mimc7_perm_lazy<false>(xs[i], r, c);
    return r;
}

// a note's commitment MultiMiMC7(m, KEY): key 0 is the transfer statement's (nullifier, secret, token, amount), key 4 the owned
// transfer statement's (owner, blinding, token, amount); NOTE_LABELED_KEY the owned labeled note's leaf
template <uint32_t KEY = 0, class CFn>
OG_HD Fr note_commitment(const Fr m[4], CFn c) {
    if (KEY == NOTE_LABELED_KEY) return note_labeled_leaf(m, c);
    const Fr k = Fr::from_u32(KEY);
    Fr r = KEY == 0 ? m[0] + mimc7_perm_lazy<true>(m[0], k, c) : k + m[0] + mimc7_perm_lazy<false>(m[0], k, c);
    for (int i = 1; i < 4; i++) r = r + m[i] + mimc7_perm_lazy<false>(m[i], r, c);
    return r;
}

OG_HD void note_store_word(uint32_t* w, const Fr& v) { v.to_canonical(w); }

// one note to the compressed key (pk_x, pk_odd) under ephemeral e; writes the record and the commitment under KEY when the
// status is NOTE_ENC_OK and zeros otherwise
template <uint32_t KEY = 0, class CFn>
OG_HD uint8_t note_encrypt_one(const Fr& pk_x, bool pk_odd, const Fr m[4], const Fr& e, const BjjBase& base, CFn c,
                               uint32_t rec[NOTE_RECORD_WORDS], Fr* cm) {
    const Fr A = bjj_a(), D = bjj_d();
    for (uint32_t i = 0; i < NOTE_RECORD_WORDS; i++) rec[i] = 0;
    *cm = Fr::zero();
    Fr vy, vx8, vy8;
    if (!bjj_decompress(&vy, &pk_x, pk_odd)) return NOTE_ENC_BAD_KEY;
    note_clear_cofactor(&vx8, &vy8, pk_x, vy);
    if (bjj_is_identity(vx8, vy8)) return NOTE_ENC_BAD_KEY;
    Fr ex, ey;
    bjj_to_pub(&ex, &ey, &base, &e);                   // E = e BASE; BASE has order l, so E = O iff e = 0 mod l
    if (bjj_is_identity(ex, ey)) return NOTE_ENC_BAD_EPHEMERAL;
    BjjPoint vp{vx8, vy8, Fr::one()}, s;
    bjj_mul(&s, &vp, &e, &A, &D);
    Fr sx, sy, pad[4];
    bjj_to_affine(&sx, &sy, &s);
    note_pads(pad, sx, sy, c);
    note_store_word(rec, ex);
    if (fr_is_odd(ey)) rec[7] |= 0x80000000u;
    for (int i = 0; i < 4; i++) note_store_word(rec + 8 * (i + 1), m[i] + pad[i]);
    *cm = note_commitment<KEY>(m, c);
    return NOTE_ENC_OK;
}

// the per-record half of a scan: false if the record is malformed (E.x >= r or bit 254 set, a c_i or the commitment >= r,
// E does not decompress, 8 E = O); else E' = affine(8 E)
OG_HD bool note_prepare_one(const uint32_t* rec, const uint32_t* cm, Fr* epx, Fr* epy) {
    uint32_t w[8];
    for (int i = 0; i < 8; i++) w[i] = rec[i];
    const bool odd = w[7] >> 31;
    w[7] &= 0x7FFFFFFFu;
    if (!Fr::canonical_lt_mod(w) || !Fr::canonical_lt_mod(cm)) return false;      // r < 2^254 covers bit 254
    for (int i = 1; i <= 4; i++)
        if (!Fr::canonical_lt_mod(rec + 8 * i)) return false;
    Fr ex = Fr::from_canonical(w), ey;
    if (!bjj_decompress(&ey, &ex, odd)) return false;
    note_clear_cofactor(epx, epy, ex, ey);
    return !bjj_is_identity(*epx, *epy);
}

// v P for an affine P through a 4-bit fixed window over a table of P's first 15 multiples (the scan's multiplier: faster
// than plain double-and-add, DESIGN.md section 8): 252 doublings and at most 64 + 14 additions instead of 255 and ~128
OG_HD void note_mul_window(BjjPoint* out, const Fr& px, const Fr& py, const uint32_t v[8]) {
    const Fr A = bjj_a(), D = bjj_d();
    BjjPoint tab[15];
    tab[0] = BjjPoint{px, py, Fr::one()};
    tab[1] = tab[0];
    bjj_double(&tab[1], &A);
    for (int d = 2; d < 15; d++) { tab[d] = tab[d - 1]; bjj_add(&tab[d], &tab[0], &A, &D); }
    BjjPoint acc{Fr::zero(), Fr::one(), Fr::zero()};
    for (int w = 63; w >= 0; w--) {
        for (int j = 0; j < 4; j++) bjj_double(&acc, &A);
        const uint32_t d = (v[w >> 3] >> ((w & 7) * 4)) & 15;
        if (d) bjj_add(&acc, &tab[d - 1], &A, &D);
    }
    *out = acc;
}

// the per-(record, key) half: the note if view key v (canonical limbs) owns the prepared record, its commitment taken under KEY
template <bool WINDOW, uint32_t KEY = 0, class CFn>
OG_HD bool note_decrypt_one(const Fr& epx, const Fr& epy, const uint32_t v[8], const uint32_t* rec, const uint32_t* cm, CFn c,
                            Fr m[4]) {
    BjjPoint s;
    if (WINDOW) {
        note_mul_window(&s, epx, epy, v);
    } else {
        const Fr A = bjj_a(), D = bjj_d(), k = Fr::from_canonical(v);
        BjjPoint ep{epx, epy, Fr::one()};
        bjj_mul(&s, &ep, &k, &A, &D);
    }
    Fr sx, sy, pad[4];
    bjj_to_affine(&sx, &sy, &s);
    note_pads(pad, sx, sy, c);
    for (int i = 0; i < 4; i++) m[i] = Fr::from_canonical(rec + 8 * (i + 1)) - pad[i];
    uint32_t a[8];
    m[3].to_canonical(a);
    for (int i = KEY == NOTE_LABELED_KEY ? 3 : 2; i < 8; i++)
        if (a[i]) return false;                       // amount >= 2^64 (2^96 for a labeled word): not a note, no need to hash it
    return note_commitment<KEY>(m, c) == Fr::from_canonical(cm);
}

}  // namespace og
