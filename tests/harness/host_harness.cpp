// tests/harness/host_harness.cpp -- compiles the product's limb algorithms (fp.cuh / ec.cuh) for the
// HOST so tests can run the exact even/odd Montgomery rows and XYZZ formulas without a GPU and
// compare them with the oracle.  Test-only; the product never proves on the host.
#include "fp.cuh"
#include "ec.cuh"
#include <cstring>
using namespace og;

template <class F> static F load(const uint8_t* b) { uint32_t c[8]; memcpy(c, b, 32); return F::from_canonical(c); }
template <class F> static void store(uint8_t* b, const F& v) { uint32_t c[8]; v.to_canonical(c); memcpy(b, c, 32); }
static Fq2 load2(const uint8_t* b) { return Fq2{load<Fq>(b), load<Fq>(b + 32)}; }
static void store2(uint8_t* b, const Fq2& v) { store(b, v.c0); store(b + 32, v.c1); }
static G1Affine loadg1(const uint8_t* b) { return G1Affine{load<Fq>(b), load<Fq>(b + 32)}; }
static void storeg1(uint8_t* b, const G1Affine& p) { store(b, p.x); store(b + 32, p.y); }
static G2Affine loadg2(const uint8_t* b) { return G2Affine{load2(b), load2(b + 64)}; }
static void storeg2(uint8_t* b, const G2Affine& p) { store2(b, p.x); store2(b + 64, p.y); }

extern "C" {
#define BINOP(name, F, expr) \
    void name(const uint8_t* a, const uint8_t* b, uint8_t* out, uint64_t n) { \
        for (uint64_t i = 0; i < n; i++) { F x = load<F>(a + 32 * i), y = load<F>(b + 32 * i); store(out + 32 * i, expr); } }
BINOP(ht_fq_mul, Fq, x * y)
BINOP(ht_fq_add, Fq, x + y)
BINOP(ht_fq_sub, Fq, x - y)
BINOP(ht_fr_mul, Fr, x * y)
BINOP(ht_fr_add, Fr, x + y)
BINOP(ht_fr_sub, Fr, x - y)
void ht_fq_inv(const uint8_t* a, uint8_t* out, uint64_t n) { for (uint64_t i = 0; i < n; i++) store(out + 32 * i, load<Fq>(a + 32 * i).inv()); }
void ht_fr_inv(const uint8_t* a, uint8_t* out, uint64_t n) { for (uint64_t i = 0; i < n; i++) store(out + 32 * i, load<Fr>(a + 32 * i).inv()); }
void ht_fq2_mul(const uint8_t* a, const uint8_t* b, uint8_t* out) { store2(out, load2(a) * load2(b)); }
void ht_fq2_sqr(const uint8_t* a, uint8_t* out) { store2(out, load2(a).sqr()); }
void ht_fq2_inv(const uint8_t* a, uint8_t* out) { store2(out, load2(a).inv()); }

void ht_g1_mul(const uint8_t* p, const uint8_t* k, uint8_t* out) { uint32_t s[8]; memcpy(s, k, 32); storeg1(out, G1XYZZ::mul(loadg1(p), s).to_affine()); }
void ht_g2_mul(const uint8_t* p, const uint8_t* k, uint8_t* out) { uint32_t s[8]; memcpy(s, k, 32); storeg2(out, G2XYZZ::mul(loadg2(p), s).to_affine()); }
// sum of n affine points, through madd (mode 0) or through XYZZ+XYZZ add of lifted points (mode 1)
void ht_g1_sum(const uint8_t* pts, uint64_t n, int mode, uint8_t* out) {
    G1XYZZ acc = G1XYZZ::inf();
    for (uint64_t i = 0; i < n; i++) {
        G1Affine q = loadg1(pts + 64 * i);
        if (mode == 0) acc.madd(q);
        else { G1XYZZ t = G1XYZZ::from_affine(q); t = t.dbl(); t.madd(q.neg()); acc.add(t); }  // 2q - q
    }
    storeg1(out, acc.to_affine());
}
void ht_g2_sum(const uint8_t* pts, uint64_t n, int mode, uint8_t* out) {
    G2XYZZ acc = G2XYZZ::inf();
    for (uint64_t i = 0; i < n; i++) {
        G2Affine q = loadg2(pts + 128 * i);
        if (mode == 0) acc.madd(q);
        else { G2XYZZ t = G2XYZZ::from_affine(q); t = t.dbl(); t.madd(q.neg()); acc.add(t); }
    }
    storeg2(out, acc.to_affine());
}
}

// ---- BabyJubJub verification core (bjj_core.cuh) on the host, placeholder-product hash -------------------
#include <vector>
#include "bjj_core.cuh"
extern "C" void ht_bjj_verify(const uint8_t* pk_x, const uint8_t* pk_odd, const uint8_t* msgs, const uint8_t* sigs, uint32_t n,
                              const uint8_t* base_xy, uint8_t* out) {
    Fr bx = load<Fr>(base_xy), by = load<Fr>(base_xy + 32);
    for (uint32_t i = 0; i < n; i++) {
        out[i] = bjj_verify_one(load<Fr>(pk_x + 32 * i), pk_odd[i] != 0, load<Fr>(msgs + 32 * i), load<Fr>(sigs + 96 * i),
                                load<Fr>(sigs + 96 * i + 32), load<Fr>(sigs + 96 * i + 64), BjjBase{bx, by, nullptr},
                                [](const Fr* in) { return in[0] * in[1] * in[2] * in[3] * in[4]; });
    }
}

// PrivateKey::to_pub + sign (bjj_core.cuh: bjj_sign_one) on the host, placeholder-product hash; and its integer step alone
extern "C" void ht_bjj_sign(const uint8_t* sks, const uint8_t* rnds, const uint8_t* msgs, uint32_t n, const uint8_t* base_xy,
                            uint8_t* pk_x, uint8_t* pk_odd, uint8_t* sigs, uint8_t* status) {
    Fr bx = load<Fr>(base_xy), by = load<Fr>(base_xy + 32);
    for (uint32_t i = 0; i < n; i++) {
        Fr px, rx, ry, s;
        bool odd;
        status[i] = bjj_sign_one(load<Fr>(sks + 32 * i), load<Fr>(rnds + 32 * i), load<Fr>(msgs + 32 * i), BjjBase{bx, by, nullptr},
                                 [](const Fr* in) { return in[0] * in[1]; },
                                 [](const Fr* in) { return in[0] * in[1] * in[2] * in[3] * in[4]; }, &px, &odd, &rx, &ry, &s);
        store(pk_x + 32 * i, px); pk_odd[i] = odd ? 1 : 0;
        store(sigs + 96 * i, rx); store(sigs + 96 * i + 32, ry); store(sigs + 96 * i + 64, s);
    }
}
// k * BASE through the window table (built here with the plain multiplier) against plain double-and-add; 1 = all equal
extern "C" int ht_bjj_table_mul_matches(const uint8_t* ks, uint32_t n, const uint8_t* base_xy) {
    const Fr A = bjj_a(), D = bjj_d();
    Fr bx = load<Fr>(base_xy), by = load<Fr>(base_xy + 32);
    std::vector<Fr> tab(2 * 64 * 15);
    BjjPoint b{bx, by, Fr::one()};
    for (int w = 0; w < 64; w++) {
        Fr x, y;
        bjj_to_affine(&x, &y, &b);
        BjjPoint base{x, y, Fr::one()}, acc{Fr::zero(), Fr::one(), Fr::zero()};
        for (int d = 1; d < 16; d++) {
            bjj_add(&acc, &base, &A, &D);
            bjj_to_affine(&tab[2 * (w * 15 + d - 1)], &tab[2 * (w * 15 + d - 1) + 1], &acc);
        }
        for (int k = 0; k < 4; k++) bjj_double(&b, &A);
    }
    for (uint32_t i = 0; i < n; i++) {
        Fr k = load<Fr>(ks + 32 * i), x1, y1, x2, y2;
        BjjPoint p1, p2;
        BjjBase plain{bx, by, nullptr}, table{bx, by, tab.data()};
        bjj_mul_base(&p1, &plain, &k, &A, &D);
        bjj_mul_base(&p2, &table, &k, &A, &D);
        bjj_to_affine(&x1, &y1, &p1); bjj_to_affine(&x2, &y2, &p2);
        if (x1 != x2 || y1 != y2) return 0;
    }
    return 1;
}
extern "C" void ht_bjj_s_mod_order(const uint8_t* r, const uint8_t* h, const uint8_t* a, uint8_t* out, uint32_t n) {
    for (uint32_t i = 0; i < n; i++) {
        uint32_t rc[8], hc[8], ac[8], sc[8];
        memcpy(rc, r + 32 * i, 32); memcpy(hc, h + 32 * i, 32); memcpy(ac, a + 32 * i, 32);
        bjj_s_mod_order(sc, rc, hc, ac);
        memcpy(out + 32 * i, sc, 32);
    }
}

// ---- wide products / separate reduction (fp.cuh: mul_wide, sqr_wide, mont_reduce_wide) ----------------------
extern "C" void ht_wide(const uint8_t* a, const uint8_t* b, uint8_t* mul32, uint8_t* sqr32, uint64_t n) {
    for (uint64_t i = 0; i < n; i++) {
        Fq x = load<Fq>(a + 32 * i), y = load<Fq>(b + 32 * i), r;
        uint32_t T[16];
        mul_wide(T, x.l, y.l); mont_reduce_wide<FqParams>(r.l, T); store(mul32 + 32 * i, r);
        sqr_wide(T, x.l); mont_reduce_wide<FqParams>(r.l, T); store(sqr32 + 32 * i, r);
    }
}

// ---- lazy-reduction chain (mimc_core.cuh): the very code the MiMC7 kernels run, on the host ------------------------
#include "host_math.hpp"
#include "mimc_core.cuh"
extern "C" void ht_mimc7_hash2_lazy(const uint8_t* l, const uint8_t* r, uint8_t* out, uint64_t n) {
    static Fr c[MIMC_ROUNDS];
    static bool init = false;
    if (!init) { mimc7_round_constants(c); init = true; }
    for (uint64_t i = 0; i < n; i++)
        store(out + 32 * i, mimc7_hash2_lazy(load<Fr>(l + 32 * i), load<Fr>(r + 32 * i), [&](int k) { return c[k]; }));
}
// raw lazy ops on operands given as 256-bit integers < 2p in MONTGOMERY form (no conversion): out = raw limbs of the result.
// op 0: mul_lazy, 1: sqr_lazy (of a), 2: add_raw + reduce_4p_to_2p
extern "C" void ht_fr_lazy_raw(int op, const uint8_t* a, const uint8_t* b, uint8_t* out, uint64_t n) {
    for (uint64_t i = 0; i < n; i++) {
        Fr x, y, z;
        memcpy(x.l, a + 32 * i, 32); memcpy(y.l, b + 32 * i, 32);
        z = op == 0 ? Fr::mul_lazy(x, y) : (op == 1 ? x.sqr_lazy() : Fr::add_raw(x, y).reduce_4p_to_2p());
        memcpy(out + 32 * i, z.l, 32);
    }
}

// the same for Fq, numbered as og_field_probe_raw's G1 unit: op 0 a * b, 1 a.sqr() (the bucket kernel's squarer), 2 a - b, 3 a.dbl()
extern "C" void ht_fq_raw(int op, const uint8_t* a, const uint8_t* b, uint8_t* out, uint64_t n) {
    for (uint64_t i = 0; i < n; i++) {
        Fq x, y, z;
        memcpy(x.l, a + 32 * i, 32); memcpy(y.l, b + 32 * i, 32);
        z = op == 0 ? x * y : op == 1 ? x.sqr() : op == 2 ? x - y : x.dbl();
        memcpy(out + 32 * i, z.l, 32);
    }
}

// ---- GLV decomposition (glv.cuh): out = |k1| (32 B) | |k2| (32 B) | sign bits (1 B: bit 0 = k1 < 0, bit 1 = k2 < 0) per scalar
#include "glv.cuh"
extern "C" void ht_glv_decompose(const uint8_t* ks, uint8_t* out, uint64_t n) {
    for (uint64_t i = 0; i < n; i++) {
        uint32_t k[8], a[8], b[8];
        bool n1, n2;
        memcpy(k, ks + 32 * i, 32);
        glv_decompose(k, a, n1, b, n2);
        memcpy(out + 65 * i, a, 32); memcpy(out + 65 * i + 32, b, 32);
        out[65 * i + 64] = (uint8_t)((n1 ? 1 : 0) | (n2 ? 2 : 0));
    }
}
extern "C" void ht_glv_beta(uint8_t* out) { for (int i = 0; i < 8; i++) { uint32_t v = Glv::beta(i); memcpy(out + 4 * i, &v, 4); } }
