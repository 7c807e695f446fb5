// owshen_b200/csrc/bjj_core.cuh -- BabyJubJub point arithmetic and the per-signature verification logic,
// host+device so tests can run the exact code without a GPU.  Follows the reference's
// /root/reference/src/blockchain/tx/owshen_airdrop/babyjubjub/mod.rs (line numbers at each function).
#pragma once
#include "fp.cuh"

#if defined(__CUDA_ARCH__)
#define OG_BJJ_FN static __device__ __noinline__
#else
#define OG_BJJ_FN static inline
#endif

namespace og {

struct BjjPoint { Fr x, y, z; };     // z == 0: the reference's "empty accumulator" sentinel

OG_HD Fr bjj_a() { return Fr::from_u32(168700); }
OG_HD Fr bjj_d() { return Fr::from_u32(168696); }

OG_BJJ_FN void bjj_double(BjjPoint* p, const Fr* A) {
    if (p->z.is_zero()) return;
    Fr b = (p->x + p->y).sqr(), c = p->x.sqr(), d = p->y.sqr();
    Fr e = *A * c, f = e + d, h = p->z.sqr();
    Fr j = f - h.dbl();
    p->x = (b - c - d) * j;
    p->y = f * (e - d);
    p->z = f * j;
}

// unified addition (complete on this curve: a is a square, d is not), so the reference's
// "equal points -> double" branch needs no special case
OG_BJJ_FN void bjj_add(BjjPoint* p, const BjjPoint* q, const Fr* A, const Fr* D) {
    if (p->z.is_zero()) { *p = *q; return; }
    if (q->z.is_zero()) return;
    Fr a = p->z * q->z, b = a.sqr(), c = p->x * q->x, d = p->y * q->y;
    Fr e = *D * c * d, f = b - e, g = b + e;
    Fr x3 = a * f * ((p->x + p->y) * (q->x + q->y) - c - d);
    Fr y3 = a * g * (d - *A * c);
    p->x = x3; p->y = y3; p->z = f * g;
}

OG_BJJ_FN void bjj_mul(BjjPoint* out, const BjjPoint* base, const Fr* k, const Fr* A, const Fr* D) {
    uint32_t s[8];
    k->to_canonical(s);
    BjjPoint acc{Fr::zero(), Fr::one(), Fr::zero()};
    for (int i = 255; i >= 0; i--) {
        bjj_double(&acc, A);
        if ((s[i >> 5] >> (i & 31)) & 1) bjj_add(&acc, base, A, D);
    }
    *out = acc;
}

OG_HD bool bjj_on_curve(const Fr& x, const Fr& y, const Fr& A, const Fr& D) {
    Fr xx = x.sqr(), yy = y.sqr();
    return yy + A * xx == Fr::one() + D * xx * yy;
}

// Tonelli-Shanks (r - 1 = 2^28 t, non-residue 7); false if a is a non-residue
OG_BJJ_FN bool fr_sqrt(Fr* out, const Fr* a) {
    if (a->is_zero()) { *out = *a; return true; }
    // t = (r - 1) >> 28
    uint32_t e[8];
#pragma unroll
    for (int i = 0; i < 8; i++) e[i] = FrParams::mod(i);
    e[0] -= 1;
    uint32_t t[8];
    for (int i = 0; i < 8; i++) t[i] = (e[i] >> 28) | (i < 7 ? e[i + 1] << 4 : 0);
    uint32_t half[8];                                  // (t + 1) / 2 ; t is odd
    {
        uint32_t c = 1;
        for (int i = 0; i < 8; i++) { uint32_t v = t[i] + c; c = (v < c) ? 1 : 0; half[i] = v; }
        for (int i = 0; i < 8; i++) half[i] = (half[i] >> 1) | (i < 7 ? half[i + 1] << 31 : 0);
    }
    Fr z = Fr::from_u32(7).pow(t);
    Fr x = a->pow(half), b = a->pow(t);
    uint32_t m = 28;
    while (b != Fr::one()) {
        uint32_t i = 0;
        Fr b2 = b;
        while (b2 != Fr::one()) { b2 = b2.sqr(); i++; if (i == m) return false; }
        Fr w = z;
        for (uint32_t k = 0; k + i + 1 < m; k++) w = w.sqr();
        x = x * w; z = w.sqr(); b = b * z; m = i;
    }
    *out = x;
    return true;
}

OG_HD bool fr_is_odd(const Fr& v) { uint32_t c[8]; v.to_canonical(c); return c[0] & 1; }


// PointCompressed::decompress (mod.rs:88-98): y of the point (x, y) whose parity is `odd`; false where the reference
// returns Err (1 - D x^2 is zero, or (1 - A x^2) / (1 - D x^2) is not a square)
OG_BJJ_FN bool bjj_decompress(Fr* y, const Fr* x, bool odd) {
    const Fr A = bjj_a(), D = bjj_d(), one = Fr::one();
    Fr xx = x->sqr();
    Fr den = one - D * xx;
    if (den.is_zero()) return false;
    Fr y2 = den.inv() * (one - A * xx);
    if (!fr_sqrt(y, &y2)) return false;
    if (fr_is_odd(*y) != odd) *y = y->neg();
    return true;
}

// status: 1 verifies, 0 does not, 2 = Err in the reference (public key does not decompress).  `h_mimc` is only
// read when hash_kind == 1 (the caller computes MultiMiMC7([R.x, R.y, pk.x, pk.y, msg]) after decompression via cb).
// fixed-base multiplication k * BASE from a table of window multiples: tab[w * 15 + d - 1] = d * 16^w * BASE (affine x, y),
// 64 additions instead of 256 doublings + ~128 additions; the additions are the reference's projective formulas
OG_BJJ_FN void bjj_mul_base_table(BjjPoint* out, const Fr* tab_xy, const Fr* k, const Fr* A, const Fr* D) {
    uint32_t s[8];
    k->to_canonical(s);
    BjjPoint acc{Fr::zero(), Fr::one(), Fr::zero()};
    for (int w = 0; w < 64; w++) {
        uint32_t d = (s[w >> 3] >> ((w & 7) * 4)) & 15;
        if (!d) continue;
        const Fr* e = tab_xy + 2 * (w * 15 + d - 1);
        BjjPoint q{e[0], e[1], Fr::one()};
        bjj_add(&acc, &q, A, D);
    }
    *out = acc;
}

// the fixed base: its coordinates and, when available, the window table (nullptr = plain double-and-add: host harness)
struct BjjBase { Fr x, y; const Fr* tab_xy; };
OG_BJJ_FN void bjj_mul_base(BjjPoint* out, const BjjBase* b, const Fr* k, const Fr* A, const Fr* D) {
    if (b->tab_xy) { bjj_mul_base_table(out, b->tab_xy, k, A, D); return; }
    BjjPoint base{b->x, b->y, Fr::one()};
    bjj_mul(out, &base, k, A, D);
}

template <class HashFn>
OG_HD uint8_t bjj_verify_one(const Fr& x, bool pk_odd, const Fr& msg, const Fr& rx, const Fr& ry, const Fr& s, const BjjBase& base,
                             HashFn hash5) {
    const Fr A = bjj_a(), D = bjj_d(), one = Fr::one();
    Fr y;
    if (!bjj_decompress(&y, &x, pk_odd)) return 2;
    // verify (mod.rs:99-115)
    if (!bjj_on_curve(x, y, A, D) || !bjj_on_curve(rx, ry, A, D)) return 0;
    Fr in[5] = {rx, ry, x, y, msg};
    Fr h = hash5(in);
    BjjPoint pk{x, y, one}, rr{rx, ry, one}, sb, ha;
    bjj_mul_base(&sb, &base, &s, &A, &D);
    bjj_mul(&ha, &pk, &h, &A, &D);
    bjj_add(&ha, &rr, &A, &D);
    // affine equality by cross-multiplication; an empty accumulator is the affine point (0, 1)
    if (sb.z.is_zero()) sb = BjjPoint{Fr::zero(), one, one};
    if (ha.z.is_zero()) ha = BjjPoint{Fr::zero(), one, one};
    bool eq = (sb.x * ha.z == ha.x * sb.z) && (sb.y * ha.z == ha.y * sb.z);
    return eq ? 1 : 0;
}

// ---- signing and key derivation (mod.rs:206-237) -----------------------------------------------------------------
// ORDER = 8 * l (mod.rs:185-188), little-endian 32-bit limbs
OG_HD uint32_t bjj_order_limb(int i) {
    constexpr uint32_t o[8] = {0xc9093788u, 0x3b94bee1u, 0xc9077053u, 0x59f76dc1u, 0x8181585du, 0xb85045b6u, 0xe131a029u, 0x30644e72u};
    return o[i];
}

// out = (r + h * a) mod ORDER on canonical integers (the reference does this in BigUint, mod.rs:224-228)
OG_BJJ_FN void bjj_s_mod_order(uint32_t* out, const uint32_t* r, const uint32_t* h, const uint32_t* a) {
    uint32_t t[17];
    for (int i = 0; i < 17; i++) t[i] = 0;
    for (int i = 0; i < 8; i++) {
        uint64_t carry = 0;
        for (int j = 0; j < 8; j++) {
            uint64_t v = (uint64_t)h[i] * a[j] + t[i + j] + carry;
            t[i + j] = (uint32_t)v; carry = v >> 32;
        }
        t[i + 8] = (uint32_t)carry;
    }
    uint64_t c = 0;
    for (int i = 0; i < 17; i++) { uint64_t v = (uint64_t)t[i] + (i < 8 ? r[i] : 0) + c; t[i] = (uint32_t)v; c = v >> 32; }
    // binary long division: rem < ORDER < 2^254 throughout, so rem * 2 + bit fits 8 limbs
    uint32_t rem[8];
    for (int i = 0; i < 8; i++) rem[i] = 0;
    for (int bit = 17 * 32 - 1; bit >= 0; bit--) {
        uint32_t in = (t[bit >> 5] >> (bit & 31)) & 1;
        for (int i = 7; i > 0; i--) rem[i] = (rem[i] << 1) | (rem[i - 1] >> 31);
        rem[0] = (rem[0] << 1) | in;
        uint32_t d[8];
        uint64_t borrow = 0;
        for (int i = 0; i < 8; i++) { uint64_t v = (uint64_t)rem[i] - bjj_order_limb(i) - borrow; d[i] = (uint32_t)v; borrow = (v >> 63) & 1; }
        if (!borrow) for (int i = 0; i < 8; i++) rem[i] = d[i];
    }
    for (int i = 0; i < 8; i++) out[i] = rem[i];
}

// the reference's to_affine (mod.rs:165-171): the empty accumulator is the affine neutral element (0, 1)
OG_BJJ_FN void bjj_to_affine(Fr* x, Fr* y, const BjjPoint* p) {
    if (p->z.is_zero()) { *x = Fr::zero(); *y = Fr::one(); return; }
    Fr zi = p->z.inv();
    *x = p->x * zi; *y = p->y * zi;
}

// PrivateKey::to_pub (mod.rs:207-209): the affine point sk BASE; the public key is its compression (x, parity of y), and
// decompressing that gives y back
OG_BJJ_FN void bjj_to_pub(Fr* x, Fr* y, const BjjBase* base, const Fr* sk) {
    const Fr A = bjj_a(), D = bjj_d();
    BjjPoint acc;
    bjj_mul_base(&acc, base, sk, &A, &D);
    bjj_to_affine(x, y, &acc);
}

// PrivateKey::to_pub + sign (mod.rs:207-237).  status 1: pk and signature written; 2: the reference returns
// Err("Invalid repr") because s >= r cannot be represented as an Fp (ORDER > r: the wart SURVEY.md 8a notes).
template <class HashFn2, class HashFn5>
OG_HD uint8_t bjj_sign_one(const Fr& sk, const Fr& randomness, const Fr& msg, const BjjBase& base, HashFn2 hash2,
                           HashFn5 hash5, Fr* pk_x, bool* pk_odd, Fr* sig_rx, Fr* sig_ry, Fr* sig_s) {
    const Fr A = bjj_a(), D = bjj_d();
    BjjPoint acc;
    Fr px, py, rx, ry;
    bjj_to_pub(&px, &py, &base, &sk);
    *pk_x = px; *pk_odd = fr_is_odd(py);
    Fr in2[2] = {randomness, msg};
    Fr r = hash2(in2);                                 // r = H(b, M)
    bjj_mul_base(&acc, &base, &r, &A, &D);                    // R = r B
    bjj_to_affine(&rx, &ry, &acc);
    Fr in5[5] = {rx, ry, px, py, msg};
    Fr h = hash5(in5);                                 // h = H(R, A, M)
    uint32_t rc[8], hc[8], ac[8], sc[8];
    r.to_canonical(rc); h.to_canonical(hc); sk.to_canonical(ac);
    bjj_s_mod_order(sc, rc, hc, ac);                   // s = (r + h a) mod ORDER
    *sig_rx = rx; *sig_ry = ry;
    if (!Fr::canonical_lt_mod(sc)) { *sig_s = Fr::zero(); return 2; }
    *sig_s = Fr::from_canonical(sc);
    return 1;
}

}  // namespace og
