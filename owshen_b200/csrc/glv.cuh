// owshen_b200/csrc/glv.cuh -- GLV decomposition of BN254 scalars for the one-shot G1 MSM (host + device).
//
// G1 has the endomorphism phi(x, y) = (beta x, y) = lambda (x, y) with beta^3 = 1 in Fq and lambda^3 = 1 in Fr, so
//     k P = k1 P + k2 phi(P),   k = k1 + k2 lambda (mod r),   |k1|, |k2| < 2^127:
// an n-point MSM with 254-bit scalars becomes a 2n-point MSM with 127-bit scalars -- the same number of bucket additions, but
// half the windows, i.e. half the bucket sets to reduce and half the ~240 sequential doublings of the final Horner, which are a
// large share of a 2^20-point MSM's time.  Public technique (Gallant-Lambert-Vanstone, CRYPTO 2001);
// not in the reference (SURVEY.md section 0).  The short lattice basis comes from the extended Euclid on (r, lambda):
//     v1 = (A1, -NB1),  v2 = (A2, A1),   a_i + b_i lambda = 0 (mod r)
// and  c1 = round(b2 k / r), c2 = round(-b1 k / r)  are taken with precomputed  G_i = round(2^256 b / r):  c = (G k + 2^255) >> 256
// (error < 1/8 of a unit, so |k1|, |k2| <= 0.625 (|a1| + |a2|) < 0.55 * 2^127).  k1 = k - c1 A1 - c2 A2,  k2 = c1 NB1 - c2 A1,
// exact integers.  tests/test_host_limbs.py checks this code against big-integer arithmetic; the GPU parity tests check the MSM.
#pragma once
#include "fp.cuh"

namespace og {

struct Glv {
    // lambda = 0xb3c4d79d41a917585bfc41088d8daaa78b17ea66b99c90dd, beta = 0x59e26bcea0d48bacd4f263f1acdb5c4f5763473177fffffe
    OG_HD static constexpr uint32_t beta(int i) {
        constexpr uint32_t m[8] = {0x77fffffeu, 0x57634731u, 0xacdb5c4fu, 0xd4f263f1u, 0xa0d48bacu, 0x59e26bceu, 0x00000000u, 0x00000000u};
        return m[i];
    }
    OG_HD static constexpr uint32_t g1(int i) { constexpr uint32_t m[3] = {0xc7e0b3d7u, 0xd91d232eu, 0x00000002u}; return m[i]; }
    OG_HD static constexpr uint32_t g2(int i) { constexpr uint32_t m[5] = {0x391eb18eu, 0x7a7bd9d4u, 0xa773d2cfu, 0x4ccef014u, 0x00000002u}; return m[i]; }
    OG_HD static constexpr uint32_t a1(int i) { constexpr uint32_t m[2] = {0x94d213e3u, 0x89d32568u}; return m[i]; }
    OG_HD static constexpr uint32_t a2(int i) { constexpr uint32_t m[4] = {0x1221250bu, 0x0be4e154u, 0xeeb859fdu, 0x6f4d8248u}; return m[i]; }
    OG_HD static constexpr uint32_t nb1(int i) { constexpr uint32_t m[4] = {0x7d4f1128u, 0x8211bbebu, 0xeeb859fcu, 0x6f4d8248u}; return m[i]; }
};

// out[0 .. no) = low `no` limbs of a[0 .. na) * b[0 .. nb)   (plain schoolbook: this runs once per scalar, not per addition)
template <class FA, class FB>
OG_HD void glv_mul(uint32_t* out, int no, FA a, int na, FB b, int nb) {
    for (int i = 0; i < no; i++) out[i] = 0;
    for (int i = 0; i < na; i++) {
        uint64_t carry = 0;
        for (int j = 0; j < nb && i + j < no; j++) {
            uint64_t t = (uint64_t)a(i) * b(j) + out[i + j] + carry;
            out[i + j] = (uint32_t)t;
            carry = t >> 32;
        }
        for (int k = i + nb; carry && k < no; k++) {
            uint64_t t = (uint64_t)out[k] + carry;
            out[k] = (uint32_t)t;
            carry = t >> 32;
        }
    }
}

// r = a - b mod 2^256
OG_HD void glv_sub8(uint32_t* r, const uint32_t* a, const uint32_t* b) {
    uint64_t borrow = 0;
    for (int i = 0; i < 8; i++) {
        uint64_t t = (uint64_t)a[i] - b[i] - borrow;
        r[i] = (uint32_t)t;
        borrow = (t >> 32) & 1;
    }
}

// two's-complement 256-bit value -> (magnitude, sign); the magnitude is below 2^127
OG_HD bool glv_abs(uint32_t* mag8, const uint32_t* v) {
    const bool neg = v[7] >> 31;
    uint64_t carry = neg;
    for (int i = 0; i < 8; i++) {
        uint64_t t = (uint64_t)(neg ? ~v[i] : v[i]) + carry;
        mag8[i] = (uint32_t)t;
        carry = t >> 32;
    }
    return neg;
}

// k (canonical, < r) -> |k1|, |k2| as 8-limb integers (upper four limbs zero) and their signs
OG_HD void glv_decompose(const uint32_t* k, uint32_t* k1mag, bool& neg1, uint32_t* k2mag, bool& neg2) {
    auto K = [&](int i) { return k[i]; };
    uint32_t t[13], c1[5], c2[5];
    // c = (G k + 2^255) >> 256
    glv_mul(t, 11, [](int i) { return Glv::g1(i); }, 3, K, 8);
    {
        uint64_t carry = 0x80000000ull;
        for (int i = 7; i < 11; i++) { uint64_t s = (uint64_t)t[i] + carry; t[i] = (uint32_t)s; carry = s >> 32; }
    }
    c1[0] = t[8]; c1[1] = t[9]; c1[2] = t[10]; c1[3] = 0; c1[4] = 0;
    glv_mul(t, 13, [](int i) { return Glv::g2(i); }, 5, K, 8);
    {
        uint64_t carry = 0x80000000ull;
        for (int i = 7; i < 13; i++) { uint64_t s = (uint64_t)t[i] + carry; t[i] = (uint32_t)s; carry = s >> 32; }
    }
    for (int i = 0; i < 5; i++) c2[i] = t[8 + i];
    auto C1 = [&](int i) { return c1[i]; };
    auto C2 = [&](int i) { return c2[i]; };
    uint32_t p[8], q[8], v[8];
    // k1 = k - c1 A1 - c2 A2   (mod 2^256; the true value is a small signed integer)
    glv_mul(p, 8, C1, 3, [](int i) { return Glv::a1(i); }, 2);
    glv_mul(q, 8, C2, 5, [](int i) { return Glv::a2(i); }, 4);
    glv_sub8(v, k, p);
    glv_sub8(v, v, q);
    neg1 = glv_abs(k1mag, v);
    // k2 = c1 NB1 - c2 A1
    glv_mul(p, 8, C1, 3, [](int i) { return Glv::nb1(i); }, 4);
    glv_mul(q, 8, C2, 5, [](int i) { return Glv::a1(i); }, 2);
    glv_sub8(v, p, q);
    neg2 = glv_abs(k2mag, v);
}

}  // namespace og
