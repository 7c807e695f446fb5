// owshen_b200/csrc/pairing.cu -- host-side Groth16 verifier: optimal-ate pairing on BN254 over the
// tower Fq2 -> Fq12 = Fq2[w]/(w^6 - (9+i)), affine Miller loop on the D-type twist, generic final
// exponentiation.  og_groth16_verify is a host function by design (three pairings; SURVEY.md 8f.1);
// it shares nothing with oracle/pairing.py except the public definition of the pairing, and tests
// check that both accept/reject the same proofs.  Field arithmetic is fp.cuh compiled for the host.
#include "groth16.cuh"
#include <vector>

namespace og {

static const uint32_t FINAL_EXP[88] = {0xca86f120u, 0x86964b64u, 0xe54523a4u, 0x40a4efb7u, 0x96e84abbu, 0x837fa978u, 0xb9b2b918u, 0x361102b6u, 0xf35692dau, 0xc0de81deu, 0xa6c3c760u, 0xbe04c7e8u, 0xd570bb7fu, 0xd766f9c9u, 0x83561841u, 0xc230974du, 0xc3be69a3u, 0x5bba1668u, 0x10526294u, 0x7f3811c4u, 0xdadda71cu, 0x29baee7du, 0x145da900u, 0xbf813b8du, 0x423f9a2cu, 0x641bbadfu, 0x44eacc5eu, 0xa80bb4eau, 0x14fde37cu, 0xcd656648u, 0x580291d2u, 0x4a0364b9u, 0x0826f0ddu, 0xee93dfb1u, 0xc5514724u, 0x6b42db8du, 0x0b0f3785u, 0xbb10cf43u, 0x6f804216u, 0x40494e40u, 0xacf3aafbu, 0x55cfe107u, 0xe0ebae87u, 0x2088ec80u, 0x11a337a0u, 0x846a3ed0u, 0x1e3a5195u, 0x48a45a4au, 0xdfc50e16u, 0xe5664568u, 0x4c0cc4ebu, 0xab6a4129u, 0xd268c7dau, 0x82d0d602u, 0xed3cc48au, 0x6668449au, 0xb2015dfcu, 0x5062cd0fu, 0xb1ddb3d1u, 0x7f2940a8u, 0x2a226448u, 0x77f5b63au, 0x61e443aeu, 0xfef07813u, 0x88d5c6c8u, 0xf977870eu, 0x1f676baau, 0x790364a6u, 0xceaddea3u, 0x5887e72eu, 0xa09a1b70u, 0x1377e563u, 0x1bd8c3b2u, 0x0c54efeeu, 0xd524d8f7u, 0x3ec3d15au, 0xb2383a5du, 0xdaf15466u, 0xbb94fec0u, 0xe1e30a73u, 0x5f3f7be2u, 0x6a1c7101u, 0x6369b1ffu, 0x842d43bfu, 0x107d20bcu, 0x20fddadfu, 0x4b6dc970u, 0x0000002fu};
static const uint32_t EXP_P_MINUS_1_OVER_3[8] = {0x4829a9c2u, 0x69602eb2u, 0xcd7b4384u, 0xdd2b2385u, 0x808072c9u, 0xe81ac1e7u, 0xa065e00du, 0x10216f7bu};
static const uint32_t EXP_P_MINUS_1_OVER_2[8] = {0x6c3e7ea3u, 0x9e10460bu, 0xb438e546u, 0xcbc0b548u, 0x40c0ac2eu, 0xdc2822dbu, 0x7098d014u, 0x18322739u};
static const uint32_t FR_MODULUS[8] = {0xf0000001u, 0x43e1f593u, 0x79b97091u, 0x2833e848u, 0x8181585du, 0xb85045b6u, 0xe131a029u, 0x30644e72u};

struct Fq12 {   // sum_k c[k] w^k, w^6 = xi = 9 + i
    Fq2 c[6];
    static Fq12 one() { Fq12 r; for (int i = 0; i < 6; i++) r.c[i] = Fq2::zero(); r.c[0] = Fq2::one(); return r; }
    bool is_one() const {
        if (!(c[0] == Fq2::one())) return false;
        for (int i = 1; i < 6; i++) if (!c[i].is_zero()) return false;
        return true;
    }
};

static Fq2 xi() { return Fq2{Fq::from_u32(9), Fq::from_u32(1)}; }
static Fq2 mul_xi(const Fq2& a) {   // (a0 + a1 i)(9 + i) = (9 a0 - a1) + (a0 + 9 a1) i
    Fq n0 = a.c0.dbl().dbl().dbl() + a.c0, n1 = a.c1.dbl().dbl().dbl() + a.c1;
    return Fq2{n0 - a.c1, n1 + a.c0};
}

static Fq12 f12_mul(const Fq12& a, const Fq12& b) {
    Fq2 t[11];
    for (int i = 0; i < 11; i++) t[i] = Fq2::zero();
    for (int i = 0; i < 6; i++) {
        if (a.c[i].is_zero()) continue;
        for (int j = 0; j < 6; j++) {
            if (b.c[j].is_zero()) continue;
            t[i + j] = t[i + j] + a.c[i] * b.c[j];
        }
    }
    Fq12 r;
    for (int k = 0; k < 6; k++) r.c[k] = t[k];
    for (int k = 6; k < 11; k++) r.c[k - 6] = r.c[k - 6] + mul_xi(t[k]);
    return r;
}

static Fq12 f12_pow(const Fq12& a, const uint32_t* e, int n_limbs) {
    Fq12 acc = Fq12::one();
    bool started = false;
    for (int i = n_limbs * 32 - 1; i >= 0; i--) {
        if (started) acc = f12_mul(acc, acc);
        if ((e[i >> 5] >> (i & 31)) & 1) { acc = started ? f12_mul(acc, a) : a; started = true; }
    }
    return acc;
}

static Fq2 f2_pow(const Fq2& a, const uint32_t* e, int n_limbs) {
    Fq2 acc = Fq2::one();
    for (int i = n_limbs * 32 - 1; i >= 0; i--) {
        acc = acc.sqr();
        if ((e[i >> 5] >> (i & 31)) & 1) acc = acc * a;
    }
    return acc;
}

// line through T and Q on the twist (or the tangent at T when Q == T), evaluated at P in G1:
//   l = yP - lambda xP w + (lambda xT - yT) w^3        (up to a factor in Fq, killed by the final exponentiation)
// advances T to T + Q.  Returns false if the sum is the point at infinity (never for valid inputs).
static bool line_step(Fq12& f, G2Affine& T, const G2Affine& Q, const G1Affine& P) {
    Fq2 lambda;
    if (T.x == Q.x) {
        if (!(T.y == Q.y) || T.y.is_zero()) return false;
        Fq2 xx = T.x.sqr();
        lambda = (xx.dbl() + xx) * T.y.dbl().inv();
    } else {
        lambda = (Q.y - T.y) * (Q.x - T.x).inv();
    }
    Fq12 l;
    for (int i = 0; i < 6; i++) l.c[i] = Fq2::zero();
    l.c[0] = Fq2{P.y, Fq::zero()};
    l.c[1] = lambda.mul_fq(P.x).neg();
    l.c[3] = lambda * T.x - T.y;
    f = f12_mul(f, l);
    Fq2 x3 = lambda.sqr() - T.x - Q.x;
    Fq2 y3 = lambda * (T.x - x3) - T.y;
    T = G2Affine{x3, y3};
    return true;
}

static bool miller_loop(Fq12& acc, const G2Affine& Q, const G1Affine& P) {
    if (Q.is_inf() || P.is_inf()) return true;     // contributes 1
    Fq12 f = Fq12::one();
    // 6u + 2 = 29793968203157093288 = 0x1_9d797039_be763ba8
    const uint64_t lo = 0x9d797039be763ba8ull;
    G2Affine T = Q;
    for (int i = 63; i >= 0; i--) {
        f = f12_mul(f, f);
        G2Affine Tc = T;
        if (!line_step(f, T, Tc, P)) return false;
        if ((lo >> i) & 1) { if (!line_step(f, T, Q, P)) return false; }
    }
    Fq2 gx = f2_pow(xi(), EXP_P_MINUS_1_OVER_3, 8), gy = f2_pow(xi(), EXP_P_MINUS_1_OVER_2, 8);
    G2Affine Q1{Q.x.conj() * gx, Q.y.conj() * gy};
    G2Affine Q2{Q1.x.conj() * gx, Q1.y.conj() * gy};
    Q2.y = Q2.y.neg();
    if (!line_step(f, T, Q1, P)) return false;
    // last line: only the value is needed; the sum may be infinity in principle, so evaluate without advancing rules
    G2Affine Tl = T;
    if (!line_step(f, Tl, Q2, P)) return false;
    acc = f12_mul(acc, f);
    return true;
}

static bool g1_on_curve(const G1Affine& p) {
    if (p.is_inf()) return true;
    return p.y.sqr() == p.x.sqr() * p.x + Fq::from_u32(3);
}
static bool g2_on_curve(const G2Affine& p) {
    if (p.is_inf()) return true;
    Fq2 b = Fq2{Fq::from_u32(3), Fq::zero()} * xi().inv();
    return p.y.sqr() == p.x.sqr() * p.x + b;
}
static bool g2_in_subgroup(const G2Affine& p) { return G2XYZZ::mul(p, FR_MODULUS).is_inf(); }

bool load_g1(G1Affine& p, const uint8_t* b) { return host_load(p.x, b) && host_load(p.y, b + 32) && g1_on_curve(p); }
bool load_g2(G2Affine& p, const uint8_t* b) {
    return host_load(p.x.c0, b) && host_load(p.x.c1, b + 32) && host_load(p.y.c0, b + 64) && host_load(p.y.c1, b + 96) &&
           g2_on_curve(p) && g2_in_subgroup(p);
}

// prod_k e(P_k, Q_k) == 1: one Miller loop per pair, one final exponentiation
bool pairing_product_is_one(const G1Affine* P, const G2Affine* Q, int n) {
    Fq12 f = Fq12::one();
    for (int k = 0; k < n; k++)
        if (!miller_loop(f, Q[k], P[k])) return false;
    return f12_pow(f, FINAL_EXP, 88).is_one();
}

int32_t groth16_verify_host(const uint8_t* vk, uint64_t vk_len, const uint8_t* pub, uint32_t n_pub, const uint8_t* proof) {
    if (vk_len < 12 || memcmp(vk, "OGVK", 4) != 0) return OG_E_ENCODING;
    uint32_t ver, vk_pub;
    memcpy(&ver, vk + 4, 4); memcpy(&vk_pub, vk + 8, 4);
    if (ver != 1 || vk_pub != n_pub || n_pub > (1u << 16)) return OG_E_ENCODING;      // bound first: n_pub + 1 must not wrap
    if (vk_len != 12 + 64 + 128 * 3 + 64ull * ((uint64_t)n_pub + 1)) return OG_E_ENCODING;
    G1Affine alpha1, A, C;
    G2Affine beta2, gamma2, delta2, B;
    const uint8_t* q = vk + 12;
    if (!load_g1(alpha1, q) || !load_g2(beta2, q + 64) || !load_g2(gamma2, q + 192) || !load_g2(delta2, q + 320)) return OG_E_ENCODING;
    const uint8_t* ic = q + 448;
    if (!load_g1(A, proof) || !load_g2(B, proof + 64) || !load_g1(C, proof + 192)) return OG_E_ENCODING;
    if (A.is_inf() || B.is_inf() || C.is_inf()) return OG_E_VERIFY;
    G1Affine ic0;
    if (!load_g1(ic0, ic)) return OG_E_ENCODING;
    G1XYZZ acc = G1XYZZ::from_affine(ic0);
    for (uint32_t i = 0; i < n_pub; i++) {
        G1Affine pt;
        if (!load_g1(pt, ic + 64ull * (i + 1))) return OG_E_ENCODING;
        uint32_t k[8];
        memcpy(k, pub + 32ull * i, 32);
        if (!Fr::canonical_lt_mod(k)) return OG_E_ENCODING;
        G1XYZZ t = G1XYZZ::mul(pt, k);
        acc.add(t);
    }
    G1Affine X = acc.to_affine();
    // e(-A, B) e(alpha, beta) e(X, gamma) e(C, delta) == 1
    const G1Affine P[4] = {A.neg(), alpha1, X, C};
    const G2Affine Q[4] = {B, beta2, gamma2, delta2};
    return pairing_product_is_one(P, Q, 4) ? OG_OK : OG_E_VERIFY;
}

}  // namespace og
