// tests/harness/g1_lazy_harness.cpp -- the lazily reduced Fq arithmetic of fp.cuh and the G1 mixed addition of ec.cuh
// (g1_madd_lazy, the body of the G1 bucket accumulation) compiled for the HOST, so tests can drive them with operands at the
// edges of [0, 2p) and with accumulators in non-canonical form.  Test-only.
#include "fp.cuh"
#include "ec.cuh"
#include <cstring>
using namespace og;

static Fq raw1(const uint8_t* b) { Fq v; memcpy(v.l, b, 32); return v; }
static void put1(uint8_t* b, const Fq& v) { memcpy(b, v.l, 32); }
static Fq load(const uint8_t* b) { uint32_t c[8]; memcpy(c, b, 32); return Fq::from_canonical(c); }
static void store(uint8_t* b, const Fq& v) { uint32_t c[8]; v.to_canonical(c); memcpy(b, c, 32); }

struct HostAcc {                         // the accumulator's four coordinates, as the kernel's shared-memory slots hold them
    Fq* c;
    Fq ld(int i) const { return c[i]; }
    void st(int i, const Fq& v) const { c[i] = v; }
};

extern "C" {
// raw Montgomery limbs in, raw limbs out (no conversion, no reduction), 32 bytes per operand.  The numbering is
// og_field_probe_raw's for the G1 unit: 0 a * b, 1 a^2, 2 a - b, 3 a + a (canonical forms), 8 mul_lazy, 9 sqr_lazy, 10 add_lazy,
// 11 sub_lazy, 12 canonical(a), 13 is_zero_lazy(a) (1 or 0 in limb 0), 14 mul_sum_lazy(a, a, 2p - b, 2p - b)
void hl_fq_op(int op, const uint8_t* a, const uint8_t* b, uint8_t* out, uint64_t n) {
    for (uint64_t i = 0; i < n; i++) {
        Fq x = raw1(a + 32 * i), y = raw1(b + 32 * i), z;
        switch (op) {
            case 0: z = x * y; break;
            case 1: z = x.sqr(); break;
            case 2: z = x - y; break;
            case 3: z = x.dbl(); break;
            case 8: z = Fq::mul_lazy(x, y); break;
            case 9: z = fq_sqr_lazy(x); break;
            case 10: z = Fq::add_lazy(x, y); break;
            case 11: z = Fq::sub_lazy(x, y); break;
            case 12: z = x.canonical(); break;
            case 13: z = Fq::zero(); z.l[0] = x.is_zero_lazy() ? 1u : 0u; break;
            default: { const Fq v = y.neg_raw(); z = Fq::mul_sum_lazy(x, x, v, v); break; }
        }
        put1(out + 32 * i, z);
    }
}

// (a b + c d) with one reduction, four raw operands per element (the general form of op 14)
void hl_fq_mul_sum(const uint8_t* a, const uint8_t* b, const uint8_t* c, const uint8_t* d, uint8_t* out, uint64_t n) {
    for (uint64_t i = 0; i < n; i++)
        put1(out + 32 * i, Fq::mul_sum_lazy(raw1(a + 32 * i), raw1(b + 32 * i), raw1(c + 32 * i), raw1(d + 32 * i)));
}

// The G1 bucket accumulation of k_bucket_acc_sm1 on the host: acc (x, y, zz, zzz as raw lazy limbs, 128 bytes; acc_inf != 0:
// the point at infinity) += the n affine points (canonical bytes, all-zero = infinity), one g1_madd_lazy per finite point.
// out: the affine sum (canonical bytes, all-zero = infinity); out_raw: the accumulator's final raw limbs (128 bytes).
void hl_g1_bucket(const uint8_t* acc, int acc_inf, const uint8_t* pts, uint64_t n, uint8_t* out, uint8_t* out_raw) {
    Fq c[4];
    for (int k = 0; k < 4; k++) c[k] = raw1(acc + 32 * k);
    HostAcc A{c};
    bool inf = acc_inf != 0;
    for (uint64_t i = 0; i < n; i++) {
        G1Affine q{load(pts + 64 * i), load(pts + 64 * i + 32)};
        if (q.is_inf()) continue;
        if (inf) { A.st(0, q.x); A.st(1, q.y); A.st(2, Fq::one()); A.st(3, Fq::one()); inf = false; continue; }
        if (!g1_madd_lazy(A, q)) inf = true;
    }
    for (int k = 0; k < 4; k++) put1(out_raw + 32 * k, c[k]);
    G1XYZZ r = inf ? G1XYZZ::inf() : G1XYZZ{c[0].canonical(), c[1].canonical(), c[2].canonical(), c[3].canonical()};
    G1Affine a = r.to_affine();
    store(out, a.x); store(out + 32, a.y);
}
}
