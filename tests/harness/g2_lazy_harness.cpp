// tests/harness/g2_lazy_harness.cpp -- the lazily reduced Fq2 arithmetic of fp.cuh and the G2 mixed addition of ec.cuh
// (g2_madd_lazy, the body of the G2 bucket accumulation) compiled for the HOST, so tests can drive them with operands at the
// edges of [0, 2p) and with accumulators in non-canonical form.  Test-only.
#include "fp.cuh"
#include "ec.cuh"
#include <cstring>
using namespace og;

static Fq2 raw2(const uint8_t* b) { Fq2 v; memcpy(v.c0.l, b, 32); memcpy(v.c1.l, b + 32, 32); return v; }
static void put2(uint8_t* b, const Fq2& v) { memcpy(b, v.c0.l, 32); memcpy(b + 32, v.c1.l, 32); }
template <class F> static F load(const uint8_t* b) { uint32_t c[8]; memcpy(c, b, 32); return F::from_canonical(c); }
template <class F> static void store(uint8_t* b, const F& v) { uint32_t c[8]; v.to_canonical(c); memcpy(b, c, 32); }
static Fq2 load2(const uint8_t* b) { return Fq2{load<Fq>(b), load<Fq>(b + 32)}; }
static void store2(uint8_t* b, const Fq2& v) { store(b, v.c0); store(b + 32, v.c1); }

struct HostAcc {                         // the accumulator's four coordinates, as the kernel's shared-memory slots hold them
    Fq2* c;
    Fq2 ld(int i) const { return c[i]; }
    void st(int i, const Fq2& v) const { c[i] = v; }
};

extern "C" {
// raw Montgomery limbs in, raw limbs out (no conversion, no reduction): op 0 mul_lazy, 1 sqr_lazy (of a), 2 add_lazy,
// 3 sub_lazy, 4 canonical (of a); 64 bytes per operand
void hl_fq2_op(int op, const uint8_t* a, const uint8_t* b, uint8_t* out, uint64_t n) {
    for (uint64_t i = 0; i < n; i++) {
        Fq2 x = raw2(a + 64 * i), y = raw2(b + 64 * i), z;
        switch (op) {
            case 0: z = fq2_mul_lazy(x, y); break;
            case 1: z = fq2_sqr_lazy(x); break;
            case 2: z = Fq2::add_lazy(x, y); break;
            case 3: z = Fq2::sub_lazy(x, y); break;
            default: z = x.canonical(); break;
        }
        put2(out + 64 * i, z);
    }
}
void hl_fq2_is_zero_lazy(const uint8_t* a, uint8_t* out, uint64_t n) {
    for (uint64_t i = 0; i < n; i++) out[i] = raw2(a + 64 * i).is_zero_lazy() ? 1 : 0;
}

// The G2 bucket accumulation of k_bucket_acc_sm on the host: acc (x, y, zz, zzz as raw lazy limbs, 256 bytes; acc_inf != 0:
// the point at infinity) += the n affine points (canonical bytes, all-zero = infinity), one g2_madd_lazy per finite point.
// out: the affine sum (canonical bytes, all-zero = infinity); out_raw: the accumulator's final raw limbs (256 bytes).
void hl_g2_bucket(const uint8_t* acc, int acc_inf, const uint8_t* pts, uint64_t n, uint8_t* out, uint8_t* out_raw) {
    Fq2 c[4];
    for (int k = 0; k < 4; k++) c[k] = raw2(acc + 64 * k);
    HostAcc A{c};
    bool inf = acc_inf != 0;
    for (uint64_t i = 0; i < n; i++) {
        G2Affine q{load2(pts + 128 * i), load2(pts + 128 * i + 64)};
        if (q.is_inf()) continue;
        if (inf) { A.st(0, q.x); A.st(1, q.y); A.st(2, Fq2::one()); A.st(3, Fq2::one()); inf = false; continue; }
        if (!g2_madd_lazy(A, q)) inf = true;
    }
    for (int k = 0; k < 4; k++) put2(out_raw + 64 * k, c[k]);
    G2XYZZ r = inf ? G2XYZZ::inf() : G2XYZZ{c[0].canonical(), c[1].canonical(), c[2].canonical(), c[3].canonical()};
    G2Affine a = r.to_affine();
    store2(out, a.x); store2(out + 64, a.y);
}
}
