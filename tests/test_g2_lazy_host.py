"""The lazily reduced Fq2 arithmetic (fp.cuh: Fq2::mul_lazy_inl, sqr_lazy_inl, add_lazy, sub_lazy) and the G2 mixed addition
the bucket accumulation runs (ec.cuh: g2_madd_lazy), compiled for the host with the PTX carry chain emulated.  Operands are
given as raw Montgomery limbs anywhere in [0, 2p), so the edges of the lazy range are reached on purpose: every result must
be congruent to the oracle's and stay below 2p, and the exceptional cases of the group law must hold when zero is held as p."""
import ctypes as C
import itertools
import os
import random
import subprocess

import pytest

from oracle import bn254 as bn

P = bn.P
RM = (1 << 256) % P
RINV = pow(RM, -1, P)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# component values at the edges of [0, 2p) (2p < 2^255, so the largest lazy values sit just below 2p, near 2^254.6)
EDGES = [0, 1, P - 1, P, P + 1, 2 * P - 1, 2 * P - 2, 1 << 254, (1 << 254) + 12345, 2 * P - (1 << 200), (1 << 256) // 5]
assert all(0 <= e < 2 * P for e in EDGES)


@pytest.fixture(scope="module")
def h(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("g2lazy") / "libg2_lazy_harness.so")      # the source tree may be read-only
    src = os.path.join(ROOT, "tests", "harness", "g2_lazy_harness.cpp")
    subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-I" + os.path.join(ROOT, "owshen_b200", "csrc"),
                    "-o", so, src], check=True)
    return C.CDLL(so)


def pack(vals):
    return b"".join(v.to_bytes(32, "little") for v in vals)


def unpack(b):
    return [int.from_bytes(b[i:i + 32], "little") for i in range(0, len(b), 32)]


def fq2_op(h, op, a, b):
    """a, b: lists of (c0, c1) raw limb values; returns the raw results"""
    out = C.create_string_buffer(64 * len(a))
    h.hl_fq2_op(op, pack([x for v in a for x in v]), pack([x for v in b for x in v]), out, C.c_uint64(len(a)))
    r = unpack(out.raw)
    return list(zip(r[0::2], r[1::2]))


def val(raw):      # the field element a raw Montgomery pair stands for
    return (raw[0] * RINV % P, raw[1] * RINV % P)


def check(results, expect):
    for r, e in zip(results, expect):
        assert r[0] < 2 * P and r[1] < 2 * P, "lazy bound"
        assert val(r) == e


def _cases(rng, n_random):
    edge_pairs = list(itertools.product(EDGES, EDGES))
    a = [x for x, _ in itertools.product(edge_pairs, edge_pairs)]
    b = [y for _, y in itertools.product(edge_pairs, edge_pairs)]
    for _ in range(n_random):
        a.append((rng.randrange(2 * P), rng.randrange(2 * P)))
        b.append((rng.randrange(2 * P), rng.randrange(2 * P)))
    return a, b


def test_lazy_fq2_product_and_squaring_at_the_edges(h):
    a, b = _cases(random.Random(11), 3000)
    check(fq2_op(h, 0, a, b), [bn.f2_mul(val(x), val(y)) for x, y in zip(a, b)])
    check(fq2_op(h, 1, a, a), [bn.f2_sqr(val(x)) for x in a])


def test_lazy_fq2_add_sub_and_canonical_at_the_edges(h):
    a, b = _cases(random.Random(12), 3000)
    check(fq2_op(h, 2, a, b), [bn.f2_add(val(x), val(y)) for x, y in zip(a, b)])
    check(fq2_op(h, 3, a, b), [bn.f2_sub(val(x), val(y)) for x, y in zip(a, b)])
    canon = fq2_op(h, 4, a, a)
    assert canon == [(x % P, y % P) for x, y in a]


def test_lazy_fq2_zero_test(h):
    vals = [(0, 0), (P, 0), (0, P), (P, P), (1, 0), (0, 1), (P + 1, P), (P - 1, 0), (2 * P - 1, P)]
    out = C.create_string_buffer(len(vals))
    h.hl_fq2_is_zero_lazy(pack([x for v in vals for x in v]), out, C.c_uint64(len(vals)))
    assert list(out.raw) == [1, 1, 1, 1, 0, 0, 0, 0, 0]


def _acc(rng, pt, shift):
    """lazy XYZZ limbs of the finite affine pt with a random z; shift adds p to every coordinate (zero held as p, others in [p, 2p))"""
    z = (rng.randrange(1, P), rng.randrange(P))
    zz = bn.f2_sqr(z)
    zzz = bn.f2_mul(zz, z)
    coords = [bn.f2_mul(pt[0], zz), bn.f2_mul(pt[1], zzz), zz, zzz]
    raw = [tuple(c * RM % P + (P if shift else 0) for c in v) for v in coords]
    return pack([x for v in raw for x in v])


def bucket(h, acc, acc_inf, pts):
    out, raw = C.create_string_buffer(128), C.create_string_buffer(256)
    enc = b"".join(bytes(128) if p is None else bn.g2_to_bytes(p) for p in pts)
    h.hl_g2_bucket(acc, acc_inf, enc, C.c_uint64(len(pts)), out, raw)
    r = unpack(raw.raw)
    assert all(x < 2 * P for x in r), "accumulator left [0, 2p)"
    return out.raw


def test_g2_mixed_add_exceptional_cases(h):
    rng = random.Random(13)
    pts = [bn.g2_mul(bn.G2_GEN, rng.randrange(1, bn.R)) for _ in range(4)]
    enc = lambda p: bytes(128) if p is None else bn.g2_to_bytes(p)
    for shift in (False, True):
        for base in pts[:2]:
            acc = _acc(rng, base, shift)
            assert bucket(h, acc, 0, [base]) == enc(bn.g2_add(base, base))                   # P + P
            assert bucket(h, acc, 0, [bn.g2_neg(base)]) == enc(None)                          # P - P
            assert bucket(h, acc, 0, [None]) == enc(base)                                     # P + infinity
            assert bucket(h, acc, 0, [bn.g2_neg(base), pts[3]]) == enc(pts[3])                # restart after infinity
            assert bucket(h, acc, 0, [pts[2], bn.g2_neg(pts[2])]) == enc(base)                # back to where it was
            assert bucket(h, acc, 0, [pts[2], base, base]) == enc(bn.g2_add(bn.g2_add(base, pts[2]), bn.g2_add(base, base)))
    acc = bytes(256)
    assert bucket(h, acc, 1, [None, pts[0], pts[0], None, pts[1]]) == enc(bn.g2_add(bn.g2_add(pts[0], pts[0]), pts[1]))


def test_g2_mixed_add_chains_against_the_oracle(h):
    rng = random.Random(14)
    pts = [bn.g2_mul(bn.G2_GEN, rng.randrange(1, bn.R)) for _ in range(6)]
    seq = [pts[0], pts[1], pts[0], None, bn.g2_neg(pts[2]), pts[3], pts[3], pts[4], bn.g2_neg(pts[4]), pts[5]] * 3
    exp = None
    for p in seq:
        exp = bn.g2_add(exp, p)
    assert bucket(h, bytes(256), 1, seq) == bn.g2_to_bytes(exp)
