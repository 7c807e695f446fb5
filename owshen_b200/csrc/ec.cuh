// owshen_b200/csrc/ec.cuh -- short-Weierstrass (a = 0) group arithmetic in extended Jacobian
// ("XYZZ") coordinates, templated on the coordinate field (Fq -> G1, Fq2 -> G2).
//
// x = X/ZZ, y = Y/ZZZ with ZZ^3 = ZZZ^2; infinity is ZZ == 0.  Affine infinity is (0, 0), which
// is off-curve because b != 0 and matches the all-zero boundary encoding (include/owshen_b200.h).
// Formulas are the public EFD ones (madd-2008-s, add-2008-s, dbl-2008-s-1, mdbl-2008-s-1) with
// every exceptional case handled, because Pippenger buckets do meet P+P, P+(-P) and infinity.
// No counterpart in the reference (SURVEY.md section 0): its only curve is BabyJubJub.
#pragma once
#include "fp.cuh"

namespace og {

template <class F>
struct Affine {
    F x, y;
    OG_HD static Affine inf() { return Affine{F::zero(), F::zero()}; }
    OG_HD bool is_inf() const { return x.is_zero() && y.is_zero(); }
    OG_HD Affine neg() const { return Affine{x, y.neg()}; }
    OG_HD bool operator==(const Affine& o) const { return x == o.x && y == o.y; }
};

template <class F>
struct XYZZ {
    F x, y, zz, zzz;

    OG_HD static XYZZ inf() { return XYZZ{F::one(), F::one(), F::zero(), F::zero()}; }
    OG_HD bool is_inf() const { return zz.is_zero(); }
    OG_HD static XYZZ from_affine(const Affine<F>& p) {
        if (p.is_inf()) return inf();
        return XYZZ{p.x, p.y, F::one(), F::one()};
    }
    OG_HD XYZZ neg() const { return XYZZ{x, y.neg(), zz, zzz}; }

    // 2 * (affine p), p finite
    OG_HD static XYZZ dbl_affine(const Affine<F>& p) {
        F u = p.y.dbl();
        F v = u.sqr();
        F w = u * v;
        F s = p.x * v;
        F xx = p.x.sqr();
        F m = xx.dbl() + xx;
        F x3 = m.sqr() - s.dbl();
        F y3 = m * (s - x3) - w * p.y;
        return XYZZ{x3, y3, v, w};
    }

    OG_HD XYZZ dbl() const {
        if (is_inf()) return *this;
        F u = y.dbl();
        F v = u.sqr();
        F w = u * v;
        F s = x * v;
        F xx = x.sqr();
        F m = xx.dbl() + xx;
        F x3 = m.sqr() - s.dbl();
        F y3 = m * (s - x3) - w * y;
        return XYZZ{x3, y3, v * zz, w * zzz};
    }

    // this += affine q   (8M + 2S in the generic case)
    OG_HD void madd(const Affine<F>& q) {
        if (q.is_inf()) return;
        if (is_inf()) { x = q.x; y = q.y; zz = F::one(); zzz = F::one(); return; }
        F u2 = q.x * zz;
        F s2 = q.y * zzz;
        F p = u2 - x;
        F r = s2 - y;
        if (p.is_zero()) {
            if (r.is_zero()) *this = dbl_affine(q);
            else *this = inf();
            return;
        }
        F pp = p.sqr();
        F ppp = p * pp;
        F q1 = x * pp;
        F x3 = r.sqr() - ppp - q1.dbl();
        y = r * (q1 - x3) - y * ppp;
        x = x3;
        zz = zz * pp;
        zzz = zzz * ppp;
    }

    // this += o   (12M + 2S in the generic case)
    OG_HD void add(const XYZZ& o) {
        if (o.is_inf()) return;
        if (is_inf()) { *this = o; return; }
        F u1 = x * o.zz;
        F u2 = o.x * zz;
        F s1 = y * o.zzz;
        F s2 = o.y * zzz;
        F p = u2 - u1;
        F r = s2 - s1;
        if (p.is_zero()) {
            if (r.is_zero()) *this = dbl();
            else *this = inf();
            return;
        }
        F pp = p.sqr();
        F ppp = p * pp;
        F q1 = u1 * pp;
        F x3 = r.sqr() - ppp - q1.dbl();
        y = r * (q1 - x3) - s1 * ppp;
        x = x3;
        zz = zz * o.zz * pp;
        zzz = zzz * o.zzz * ppp;
    }

    OG_HD Affine<F> to_affine() const {
        if (is_inf()) return Affine<F>::inf();
        F t = (zz * zzz).inv();
        return Affine<F>{x * (t * zzz), y * (t * zz)};
    }

    // k * p, k a canonical 8-limb integer (plain MSB-first double-and-add)
    OG_HD static XYZZ mul(const Affine<F>& p, const uint32_t* k) {
        XYZZ acc = inf();
        for (int i = 255; i >= 0; i--) {
            acc = acc.dbl();
            if ((k[i >> 5] >> (i & 31)) & 1) acc.madd(p);
        }
        return acc;
    }
};

// ---- G2 mixed addition over lazily reduced Fq2 (bounds at fp.cuh: Fq2::add_lazy) ---------------------------------------
// acc += q for a finite accumulator held by A (A.ld(c) / A.st(c, v), c = 0..3 for x, y, zz, zzz, every coordinate in
// [0, 2p), each loaded where the formula uses it) and a finite affine q with canonical coordinates.  Returns false when the
// sum is the point at infinity (A is then left as it was).  The formula is XYZZ::madd's; its exceptional tests ask
// "== 0 mod p", since a lazy zero is 0 or p.  Callers make the coordinates canonical (Fq2::canonical) when a point leaves.
template <class Acc>
OG_HD bool g2_madd_lazy(const Acc& A, const Affine<Fq2>& q) {
    Fq2 p = Fq2::sub_lazy(fq2_mul_lazy(q.x, A.ld(2)), A.ld(0));
    Fq2 r = Fq2::sub_lazy(fq2_mul_lazy(q.y, A.ld(3)), A.ld(1));
    if (p.is_zero_lazy()) {
        if (!r.is_zero_lazy()) return false;                  // acc == -q
        XYZZ<Fq2> d = XYZZ<Fq2>::dbl_affine(q);               // acc == q (rare): canonical values are lazy values too
        A.st(0, d.x); A.st(1, d.y); A.st(2, d.zz); A.st(3, d.zzz);
        return true;
    }
    // ordered so that few temporaries are live at a time: zz and zzz are updated as soon as pp / ppp exist
    Fq2 pp = fq2_sqr_lazy(p);
    A.st(2, fq2_mul_lazy(A.ld(2), pp));
    Fq2 ppp = fq2_mul_lazy(p, pp);
    A.st(3, fq2_mul_lazy(A.ld(3), ppp));
    Fq2 q1 = fq2_mul_lazy(A.ld(0), pp);
    Fq2 x3 = Fq2::sub_lazy(Fq2::sub_lazy(fq2_sqr_lazy(r), ppp), Fq2::add_lazy(q1, q1));
    A.st(0, x3);
    Fq2 t = fq2_mul_lazy(A.ld(1), ppp);
    A.st(1, Fq2::sub_lazy(fq2_mul_lazy(r, Fq2::sub_lazy(q1, x3)), t));
    return true;
}

// ---- G1 mixed addition over lazily reduced Fq (bounds at fp.cuh: Fq2::add_lazy) ----------------------------------------
// g2_madd_lazy's contract on Fq: acc += q for a finite accumulator held by A (every coordinate in [0, 2p)) and a finite affine q
// with canonical coordinates; false when the sum is infinity (A is then left as it was).  The squarings go through fq_sqr_lazy
// (one out-of-line copy in the G1 MSM unit); Y3 = r (q1 - x3) - Y1 ppp is one sum of two products with a single reduction.
template <class Acc>
OG_HD bool g1_madd_lazy(const Acc& A, const Affine<Fq>& q) {
    Fq p = Fq::sub_lazy(Fq::mul_lazy(q.x, A.ld(2)), A.ld(0));
    Fq r = Fq::sub_lazy(Fq::mul_lazy(q.y, A.ld(3)), A.ld(1));
    if (p.is_zero_lazy()) {
        if (!r.is_zero_lazy()) return false;                  // acc == -q
        XYZZ<Fq> d = XYZZ<Fq>::dbl_affine(q);                 // acc == q (rare): canonical values are lazy values too
        A.st(0, d.x); A.st(1, d.y); A.st(2, d.zz); A.st(3, d.zzz);
        return true;
    }
    // ordered so that few temporaries are live at a time: zz and zzz are updated as soon as pp / ppp exist
    Fq pp = fq_sqr_lazy(p);
    A.st(2, Fq::mul_lazy(A.ld(2), pp));
    Fq ppp = Fq::mul_lazy(p, pp);
    A.st(3, Fq::mul_lazy(A.ld(3), ppp));
    Fq q1 = Fq::mul_lazy(A.ld(0), pp);
    Fq x3 = Fq::sub_lazy(Fq::sub_lazy(fq_sqr_lazy(r), ppp), Fq::add_lazy(q1, q1));
    A.st(0, x3);
    A.st(1, Fq::mul_sum_lazy(r, Fq::sub_lazy(q1, x3), A.ld(1).neg_raw(), ppp));
    return true;
}

// Out-of-line copies for kernels where a group operation is not the inner loop (reductions, table
// builds, finalisation): one body per field instead of one per call site keeps ptxas time sane.
#if defined(__CUDACC__)
template <class F> __device__ __noinline__ void xyzz_add_ni(XYZZ<F>* a, const XYZZ<F>* b) { a->add(*b); }
template <class F> __device__ __noinline__ void xyzz_madd_ni(XYZZ<F>* a, const Affine<F>* b) { a->madd(*b); }
template <class F> __device__ __noinline__ void xyzz_dbl_ni(XYZZ<F>* a) { *a = a->dbl(); }
template <class F> __device__ __noinline__ void xyzz_to_affine_ni(Affine<F>* r, const XYZZ<F>* a) { *r = a->to_affine(); }
#endif

typedef Affine<Fq> G1Affine;
typedef Affine<Fq2> G2Affine;
typedef XYZZ<Fq> G1XYZZ;
typedef XYZZ<Fq2> G2XYZZ;

}  // namespace og
