"""The lazily reduced Fq arithmetic of the G1 group law (fp.cuh: Fp::mul_lazy, sqr_lazy, add_lazy, sub_lazy, neg_raw, canonical,
is_zero_lazy and the one-reduction mul_sum_lazy) and the G1 mixed addition the bucket accumulation runs (ec.cuh: g1_madd_lazy).

Host: the same source compiled for the CPU with the PTX carry chain emulated (tests/harness/g1_lazy_harness.cpp).  Operands are
raw Montgomery limbs anywhere in [0, 2p), so the edges of the lazy range are reached on purpose -- 0, p, p - 1, 2p - 1, and pairs
that drive the one-reduction sum of two products to its 8p^2 bound -- and accumulators hold p in place of 0.  Every result must
be congruent to the exact value and stay below 2p (p for the canonical forms).

GPU: og_field_probe_raw's lazy G1 ops on the device, byte for byte against the host build and against Python integers; the G1
bucket kernel (k_bucket_acc_sm1) through og_msm_bucket_sums on crafted lists where table points repeat and appear negated under
one bucket (P + P, P - P and restarts after infinity inside one accumulation); and a one-shot G1 MSM against the C oracle."""
import ctypes as C
import itertools
import os
import random
import subprocess

import pytest

from oracle import bn254 as bn
from oracle import cport

P = bn.P
RM = (1 << 256) % P
RINV = pow(RM, -1, P)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# values at the edges of [0, 2p) (2p < 2^255), and values near 0 whose 2p - b is at the top of (0, 2p]
EDGES = [0, 1, 2, P - 1, P, P + 1, 2 * P - 1, 2 * P - 2, 1 << 254, (1 << 254) + 12345, 2 * P - (1 << 200), (1 << 256) // 5,
         (1 << 32) - 1, (1 << 224) - 1]
assert all(0 <= e < 2 * P for e in EDGES)
OPS = {"mul": 0, "sqr": 1, "sub": 2, "dbl": 3, "mul_lazy": 8, "sqr_lazy": 9, "add_lazy": 10, "sub_lazy": 11, "canonical": 12,
       "is_zero_lazy": 13, "mul_sum_lazy": 14}
LAZY = ("mul_lazy", "sqr_lazy", "add_lazy", "sub_lazy", "canonical", "is_zero_lazy", "mul_sum_lazy")


@pytest.fixture(scope="module")
def h(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("g1lazy") / "libg1_lazy_harness.so")      # the source tree may be read-only
    subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-I" + os.path.join(ROOT, "owshen_b200", "csrc"),
                    "-o", so, os.path.join(ROOT, "tests", "harness", "g1_lazy_harness.cpp")], check=True)
    return C.CDLL(so)


def pack(vals):
    return b"".join(v.to_bytes(32, "little") for v in vals)


def unpack(b):
    return [int.from_bytes(b[i:i + 32], "little") for i in range(0, len(b), 32)]


def host_op(h, op, a, b):
    out = C.create_string_buffer(32 * len(a))
    h.hl_fq_op(OPS[op], pack(a), pack(b), out, C.c_uint64(len(a)))
    return out.raw


def grid(seed, bound=2 * P, n_random=3000):
    """every pair of edge values, then random pairs below bound"""
    rng = random.Random(seed)
    edges = sorted({e % bound for e in EDGES})
    a = [x for x, _ in itertools.product(edges, edges)]
    b = [y for _, y in itertools.product(edges, edges)]
    a += [rng.randrange(bound) for _ in range(n_random)]
    b += [rng.randrange(bound) for _ in range(n_random)]
    return a, b


def exact(op, x, y):
    """the value (mod p) the raw result of op must stand for, as a raw Montgomery value"""
    return {"mul": x * y * RINV, "sqr": x * x * RINV, "sub": x - y, "dbl": 2 * x, "mul_lazy": x * y * RINV, "sqr_lazy": x * x * RINV,
            "add_lazy": x + y, "sub_lazy": x - y, "canonical": x,
            "mul_sum_lazy": (x * x + (2 * P - y) ** 2) * RINV}[op] % P


def check(op, a, b, got):
    bound = P if op in ("mul", "sqr", "sub", "dbl", "canonical") else 2 * P
    if op == "is_zero_lazy":
        assert got == [int(x % P == 0) for x in a]
        return
    for x, y, r in zip(a, b, got):
        assert r < bound and r % P == exact(op, x, y), (op, hex(x), hex(y), hex(r))
    if op == "canonical":
        assert got == [x % P for x in a]


# ---- host -----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("op", LAZY)
def test_lazy_fq_ops_at_the_edges(h, op):
    a, b = grid(21 + LAZY.index(op))
    check(op, a, b, unpack(host_op(h, op, a, b)))


@pytest.mark.parametrize("op", ("mul", "sqr", "sub", "dbl"))
def test_canonical_fq_ops_keep_their_results(h, op):
    """ops 0-3 of the probe numbering are the canonical forms, specified for the operand ranges the kernels give them"""
    a, b = grid(31 + OPS[op], bound=2 * P if op in ("mul", "sqr") else P)
    check(op, a, b, unpack(host_op(h, op, a, b)))


def test_mul_sum_reaches_its_bound(h):
    """a b + c d with one reduction, with both products near 4p^2 (T near 8p^2) and c = 2p (the neg_raw of 0)"""
    rng = random.Random(41)
    top = [2 * P - 1, 2 * P - 2, 2 * P - (1 << 200), 1 << 254, 2 * P]
    quads = [q for q in itertools.product(top, repeat=4)]
    quads += [tuple(rng.randrange(2 * P + 1) for _ in range(4)) for _ in range(3000)]
    quads += [(0, 0, 0, 0), (P, P, P, P), (2 * P, 0, 2 * P, 2 * P - 1), (1, 1, 2 * P, 2 * P)]
    cols = list(zip(*quads))
    out = C.create_string_buffer(32 * len(quads))
    h.hl_fq_mul_sum(*(pack(c) for c in cols), out, C.c_uint64(len(quads)))
    assert max(x * y + z * w for x, y, z, w in quads) > 7.99 * P * P
    for (x, y, z, w), r in zip(quads, unpack(out.raw)):
        assert r < 2 * P and r % P == (x * y + z * w) * RINV % P, (hex(x), hex(y), hex(z), hex(w))


def test_lazy_fq_zero_test(h):
    vals = [0, P, 1, P - 1, P + 1, 2 * P - 1, 1 << 254]
    assert unpack(host_op(h, "is_zero_lazy", vals, vals)) == [1, 1, 0, 0, 0, 0, 0]


def _acc(rng, pt, shift):
    """lazy XYZZ limbs of the finite affine pt with a random z; shift adds p to every coordinate, so every coordinate lies in
    [p, 2p) and the differences the formula tests for zero come out as p where the canonical accumulator gives 0"""
    z = rng.randrange(1, P)
    zz = z * z % P
    zzz = zz * z % P
    coords = [pt[0] * zz % P, pt[1] * zzz % P, zz, zzz]
    return pack([c * RM % P + (P if shift else 0) for c in coords])


def bucket(h, acc, acc_inf, pts):
    out, raw = C.create_string_buffer(64), C.create_string_buffer(128)
    enc = b"".join(bytes(64) if p is None else bn.g1_to_bytes(p) for p in pts)
    h.hl_g1_bucket(acc, acc_inf, enc, C.c_uint64(len(pts)), out, raw)
    assert all(x < 2 * P for x in unpack(raw.raw)), "accumulator left [0, 2p)"
    return out.raw


def enc(p):
    return bytes(64) if p is None else bn.g1_to_bytes(p)


def test_g1_mixed_add_exceptional_cases(h):
    rng = random.Random(43)
    pts = [bn.g1_mul(bn.G1_GEN, rng.randrange(1, bn.R)) for _ in range(4)]
    for shift in (False, True):
        for base in pts[:2]:
            acc = _acc(rng, base, shift)
            assert bucket(h, acc, 0, [base]) == enc(bn.g1_add(base, base))                   # P + P
            assert bucket(h, acc, 0, [bn.g1_neg(base)]) == enc(None)                          # P - P
            assert bucket(h, acc, 0, [None]) == enc(base)                                     # P + infinity
            assert bucket(h, acc, 0, [bn.g1_neg(base), pts[3]]) == enc(pts[3])                # restart after infinity
            assert bucket(h, acc, 0, [pts[2], bn.g1_neg(pts[2])]) == enc(base)                # back to where it was
            assert bucket(h, acc, 0, [pts[2], base, base]) == enc(bn.g1_add(bn.g1_add(base, pts[2]), bn.g1_add(base, base)))
    assert bucket(h, bytes(128), 1, [None, pts[0], pts[0], None, pts[1]]) == enc(bn.g1_add(bn.g1_add(pts[0], pts[0]), pts[1]))


def test_g1_mixed_add_chains_against_the_oracle(h):
    rng = random.Random(45)
    pts = [bn.g1_mul(bn.G1_GEN, rng.randrange(1, bn.R)) for _ in range(6)]
    seq = [pts[0], pts[1], pts[0], None, bn.g1_neg(pts[2]), pts[3], pts[3], pts[4], bn.g1_neg(pts[4]), pts[5]] * 3
    exp = None
    for p in seq:
        exp = bn.g1_add(exp, p)
    assert bucket(h, bytes(128), 1, seq) == bn.g1_to_bytes(exp)
    for shift in (False, True):          # long runs from lazy accumulators
        acc = _acc(rng, pts[5], shift)
        run = [rng.choice(pts) if rng.random() < 0.8 else bn.g1_neg(rng.choice(pts)) for _ in range(200)]
        exp = pts[5]
        for p in run:
            exp = bn.g1_add(exp, p)
        assert bucket(h, acc, 0, run) == enc(exp)


# ---- GPU ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("op", LAZY)
def test_g1_unit_lazy_ops_match_host_and_integers(ctx, h, op):
    a, b = grid(51 + LAZY.index(op))
    raw = ctx.field_probe_raw("g1", op, pack(a), pack(b))
    assert raw == host_op(h, op, a, b), op
    check(op, a, b, unpack(raw))


@pytest.mark.gpu
def test_g1_bucket_kernel_meets_doubling_and_cancellation(ctx):
    """Crafted bucket lists over a small table: the same point twice in a row (P + P), a point and its negation (P - P), and
    runs that restart after infinity, all under one bucket; every bucket against the oracle's sum."""
    rng = random.Random(61)
    logs = [rng.randrange(1, bn.R) for _ in range(8)]
    table = ctx.g1_generator_mul(cport.frs(logs))
    pts = [bn.g1_from_bytes(table[64 * i:64 * i + 64]) for i in range(len(logs))]
    E = lambda i, neg=False: (i << 1) | int(neg)
    lists = [
        [E(0), E(0)],                                     # P + P as the first addition
        [E(1), E(1, True)],                               # P - P
        [E(2), E(3), E(2), E(2)],                         # a repeat after another point, then P + P on a lazy accumulator
        [E(4), E(4, True), E(5), E(5)],                   # cancel, restart, double
        [E(6), E(7), E(7, True), E(6, True)],             # back to infinity in two steps
        [E(1), E(2), E(3), E(1, True), E(2, True), E(3, True), E(0)],
        [E(i % 8, i % 3 == 0) for i in range(40)],
        [E(5)] * 9 + [E(5, True)] * 4,
    ]
    nb = len(lists)
    counts = [len(l) for l in lists]
    entries = [e for l in lists for e in l]
    tot, bk = ctx.msm_bucket_sums("g1", table, counts, entries, 1, nb, buckets=True)

    def val(e):
        return bn.g1_neg(pts[e >> 1]) if e & 1 else pts[e >> 1]
    sums = []
    for l in lists:
        s = None
        for e in l:
            s = bn.g1_add(s, val(e))
        sums.append(s)
    assert [bk[64 * b:64 * b + 64] for b in range(nb)] == [enc(s) for s in sums]
    total = None
    for b, s in enumerate(sums):
        total = bn.g1_add(total, bn.g1_mul(s, b + 1) if s is not None else None)
    assert tot == enc(total)


@pytest.mark.gpu
def test_g1_msm_one_shot_against_the_oracle(ctx):
    from tests.helpers import rand_g1
    rng = random.Random(62)
    n = 1 << 14
    pts = rand_g1(rng, n)
    sc = cport.frs([rng.randrange(bn.R) for _ in range(n)])
    assert ctx.msm_g1(pts, sc) == cport.g1_msm(pts, sc)
