"""The limb arithmetic of the two MSM units on the device, on raw Montgomery operands chosen at the edges of the lazy range.

og_field_probe_raw runs element-wise operations in msm.cu's G1 unit (Fq: the product, the out-of-line squarer fq_sqr_call of the
bucket kernel, subtraction, doubling) and in its G2 unit, which is built with -DOG_FP_MUL_CALL (the lazy Fq2 product and squaring
through fq2_mul_lazy_call / fq2_sqr_lazy_call, the canonical ones through fq2_mul_call / fq2_sqr_call, add_lazy, sub_lazy,
canonical and is_zero_lazy).  Operands are raw limbs with no conversion and no range check, so values the bucket kernels hold only
with probability ~2^-250 -- a coordinate held as p instead of 0, values just below 2p, runs of 0xffffffff limbs -- reach the PTX
carry chains on purpose.

Each result is checked twice:
  * against Python integers: congruent to the exact value, and below 2p (lazy ops) or p (canonical ops);
  * byte for byte against the host build of the same code (tests/harness/host_harness.cpp, g2_lazy_harness.cpp), where the carry
    flag is emulated.  The device runs the same algorithm, so any difference in the raw limbs is a code-generation or carry-flag
    problem even when the value is still congruent.
The CPU tests pin the host builds of the new harness entry points to Python integers on the same grids.

What this does not check: the build is whole-program, so ptxas compiles a copy of each __noinline__ function (fq_sqr_call,
fq2_mul_lazy_call, ...) into every kernel that calls it.  The probe kernels run their own copies -- the same PTX as the bucket
kernels' copies and the same launch bounds, but not necessarily the same register allocation -- so these tests check the PTX carry
chains and ptxas's code for them, not the exact SASS inside k_bucket_acc_sm1 / k_bucket_acc_sm.  The bucket kernels' own copies
are exercised through og_msm_bucket_sums (tests/test_msm_buckets.py) on canonical points."""
import ctypes as C
import itertools
import os
import random
import subprocess

import pytest

from oracle import bn254 as bn
from tests.test_g2_lazy_host import EDGES

P = bn.P
RM = (1 << 256) % P
RINV = pow(RM, -1, P)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIMBS = [0, 1, 0xFFFFFFFF, 0xFFFFFFFE, 0x80000000, 0x7FFFFFFF]       # test_host_limbs.test_field_limbs_hypothesis's limb edges


def _harness(tmp_path_factory, name):
    so = str(tmp_path_factory.mktemp(name) / f"lib{name}.so")          # the source tree may be read-only
    subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-I" + os.path.join(ROOT, "owshen_b200", "csrc"), "-o", so,
                    os.path.join(ROOT, "tests", "harness", f"{name}.cpp")], check=True)
    return C.CDLL(so)


@pytest.fixture(scope="module")
def hg1(tmp_path_factory):
    return _harness(tmp_path_factory, "host_harness")


@pytest.fixture(scope="module")
def hg2(tmp_path_factory):
    return _harness(tmp_path_factory, "g2_lazy_harness")


def pack(vals):
    return b"".join(v.to_bytes(32, "little") for v in vals)


def unpack(b):
    return [int.from_bytes(b[i:i + 32], "little") for i in range(0, len(b), 32)]


# ---- operand grids --------------------------------------------------------------------------------------------------------
def limb_values(rng, n, bound):
    """Values below bound made of the limb edges: random 8-limb words over LIMBS, and runs of 0xffffffff limbs (2^(32k) - 1, and
    the same shifted up by j limbs), reduced below bound."""
    out = [sum(rng.choice(LIMBS) << (32 * i) for i in range(8)) % bound for _ in range(n)]
    out += [((1 << (32 * k)) - 1) << (32 * j) for k in range(1, 9) for j in range(8 - k + 1)]
    out += [(1 << 255) - 1, (1 << 254) - 1, (1 << 253) - 1, 0xFFFFFFFF << 224, bound - 1, bound - 2, bound >> 1]
    return [v % bound for v in out]


def grid1(bound, seed, n_random=3000):
    """Fq operand pairs below bound: every pair of edge values, random values and the limb patterns."""
    rng = random.Random(seed)
    edges = sorted({e % bound for e in EDGES + limb_values(rng, 0, bound)})
    a = [x for x, _ in itertools.product(edges, edges)]
    b = [y for _, y in itertools.product(edges, edges)]
    lv = limb_values(rng, 300, bound)
    a += lv + [rng.randrange(bound) for _ in range(n_random)]
    b += lv[::-1] + [rng.randrange(bound) for _ in range(n_random)]
    return a, b


def grid2(bound, seed, n_random=3000):
    """Fq2 operand pairs ((c0, c1) raw limbs) below bound: EDGES^2 x EDGES^2 as the host tests use, random values and the limb
    patterns in both coordinates."""
    rng = random.Random(seed)
    edges = sorted({e % bound for e in EDGES})
    pairs = list(itertools.product(edges, edges))
    a = [x for x, _ in itertools.product(pairs, pairs)]
    b = [y for _, y in itertools.product(pairs, pairs)]
    lv = limb_values(rng, 300, bound)
    for i, v in enumerate(lv):
        a.append((v, lv[(7 * i + 3) % len(lv)])); b.append((lv[(5 * i + 1) % len(lv)], v))
    for _ in range(n_random):
        a.append((rng.randrange(bound), rng.randrange(bound))); b.append((rng.randrange(bound), rng.randrange(bound)))
    return a, b


# ---- exact values ---------------------------------------------------------------------------------------------------------
G1_OPS = ("mul", "sqr", "sub", "dbl")
G2_OPS = ("mul_lazy", "sqr_lazy", "add_lazy", "sub_lazy", "canonical", "mul", "sqr", "is_zero_lazy")
G1_BOUND = {"mul": 2 * P, "sqr": 2 * P, "sub": P, "dbl": P}            # operand range each op is specified for
G2_LAZY = {"mul_lazy", "sqr_lazy", "add_lazy", "sub_lazy"}


def g1_exact(op, x, y):
    """The raw Montgomery value r is congruent to: (product / square / difference / double of the operands' raw values)"""
    return {"mul": x * y * RINV, "sqr": x * x * RINV, "sub": x - y, "dbl": 2 * x}[op] % P


def check_g1(op, a, b, got):
    for x, y, r in zip(a, b, got):
        assert r < P and r == g1_exact(op, x, y), (op, hex(x), hex(y), hex(r))


def check_g2(op, a, b, got):
    for (x0, x1), (y0, y1), (r0, r1) in zip(a, b, got):
        if op in ("mul_lazy", "mul"):
            e = ((x0 * y0 - x1 * y1) * RINV % P, (x0 * y1 + x1 * y0) * RINV % P)
        elif op in ("sqr_lazy", "sqr"):
            e = ((x0 * x0 - x1 * x1) * RINV % P, 2 * x0 * x1 * RINV % P)
        elif op == "add_lazy":
            e = ((x0 + y0) % P, (x1 + y1) % P)
        elif op == "sub_lazy":
            e = ((x0 - y0) % P, (x1 - y1) % P)
        elif op == "canonical":
            e = (x0 % P, x1 % P)
        else:
            assert (r0, r1) == (int(x0 % P == 0 and x1 % P == 0), 0), (hex(x0), hex(x1))
            continue
        bound = 2 * P if op in G2_LAZY else P
        assert r0 < bound and r1 < bound, (op, "bound", hex(x0), hex(x1), hex(y0), hex(y1))
        assert (r0 % P, r1 % P) == e, (op, hex(x0), hex(x1), hex(y0), hex(y1))
        if op == "canonical":
            assert (r0, r1) == e


def g2_grid(op, seed):
    """Lazy ops take operands anywhere in [0, 2p); the canonical product and squaring are specified for [0, p), is_zero_lazy and
    canonical for [0, 2p)."""
    return grid2(P if op in ("mul", "sqr") else 2 * P, seed)


def host_g1(h, op, a, b):
    out = C.create_string_buffer(32 * len(a))
    h.ht_fq_raw(G1_OPS.index(op), pack(a), pack(b), out, C.c_uint64(len(a)))
    return unpack(out.raw)


def host_g2(h, op, a, b):
    n = len(a)
    ab, bb = pack([v for x in a for v in x]), pack([v for y in b for v in y])
    if op == "is_zero_lazy":
        out = C.create_string_buffer(n)
        h.hl_fq2_is_zero_lazy(ab, out, C.c_uint64(n))
        return [(z, 0) for z in out.raw]
    out = C.create_string_buffer(64 * n)
    h.hl_fq2_op(G2_OPS.index(op), ab, bb, out, C.c_uint64(n))
    r = unpack(out.raw)
    return list(zip(r[0::2], r[1::2]))


# ---- CPU: the host builds of the probe's operations against Python integers ------------------------------------------------
@pytest.mark.parametrize("op", G1_OPS)
def test_host_fq_raw_ops(hg1, op):
    a, b = grid1(G1_BOUND[op], 100 + G1_OPS.index(op), n_random=500)
    check_g1(op, a, b, host_g1(hg1, op, a, b))


@pytest.mark.parametrize("op", G2_OPS)
def test_host_fq2_raw_ops(hg2, op):
    a, b = g2_grid(op, 200 + G2_OPS.index(op))
    a, b = a[::7] + a[-800:], b[::7] + b[-800:]
    check_g2(op, a, b, host_g2(hg2, op, a, b))


def test_grids_reach_the_edges():
    """The grids hold what the docstring claims: p itself (a zero held as p), values just below 2p, and whole words of
    0xffffffff limbs."""
    a, _ = grid1(2 * P, 1)
    assert P in a and 2 * P - 1 in a and 2 * P - 2 in a and 0 in a and (1 << 224) - 1 in a
    a, _ = grid2(2 * P, 1)
    comps = {v for x in a for v in x}
    assert {0, P, 2 * P - 1, (1 << 64) - 1, ((1 << 128) - 1) << 96} <= comps
    assert (P, 0) in a and (0, P) in a and (P, P) in a
    a, _ = grid2(P, 1)
    assert max(v for x in a for v in x) < P


# ---- GPU: the device against both -------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("op", G1_OPS)
def test_g1_unit_raw_ops_match_host_and_integers(ctx, hg1, op):
    a, b = grid1(G1_BOUND[op], 300 + G1_OPS.index(op))
    raw = ctx.field_probe_raw("g1", op, pack(a), pack(b))
    got = unpack(raw)
    assert raw == pack(host_g1(hg1, op, a, b)), op
    check_g1(op, a, b, got)


@pytest.mark.gpu
@pytest.mark.parametrize("op", G2_OPS)
def test_g2_unit_raw_ops_match_host_and_integers(ctx, hg2, op):
    a, b = g2_grid(op, 400 + G2_OPS.index(op))
    raw = ctx.field_probe_raw("g2", op, pack([v for x in a for v in x]), pack([v for y in b for v in y]))
    r = unpack(raw)
    got = list(zip(r[0::2], r[1::2]))
    host = host_g2(hg2, op, a, b)
    if op == "is_zero_lazy":
        assert got == host
    else:
        assert raw == pack([v for x in host for v in x]), op
    check_g2(op, a, b, got)


@pytest.mark.gpu
def test_field_probe_argument_errors(ctx):
    from owshen_b200 import api
    n0 = ctx.launch_count
    one = bytes(64)
    out = C.create_string_buffer(64)
    for unit, op in ((0, 4), (0, -1), (1, 8), (2, 0), (-1, 0)):
        assert api.lib().og_field_probe_raw(ctx._h, unit, op, one, one, 1, out) == api.OG_E_INVALID, (unit, op)
    assert ctx.launch_count == n0
    assert ctx.field_probe_raw("g2", "mul", b"", b"") == b""
    assert ctx.launch_count == n0
