"""The two-phase setup ceremony (DESIGN.md section 4b).  CPU: the identities key derivation rests on, and the pure-Python
spec (tests/ceremony_spec.py) against oracle.groth16.setup.  GPU: the point kernels, the accumulator bytes against the spec
and the golden, verification of honest and tampered updates, and keys byte-identical to og_groth16_setup with
tau = prod t, alpha = prod a, beta = prod b, gamma = 1, delta = prod d."""
import json
import os
import random

import pytest

import owshen_b200 as ob
from owshen_b200 import api
from oracle import bn254 as bn
from oracle import groth16 as g16
from oracle.ntt import ntt
from tests import ceremony_spec as spec
from tests.test_r1cs_setup import rand_circuit

R = bn.R
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "ceremony_vectors.json")


def prod(xs):
    p = 1
    for x in xs:
        p = p * x % R
    return p


# ---- CPU ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("log_m", [1, 2, 3, 5])
def test_lagrange_basis_is_inverse_ntt_of_powers(log_m):
    tau = random.Random(log_m).randrange(2, R)
    m = 1 << log_m
    assert ntt([pow(tau, i, R) for i in range(m)], inverse=True) == g16.lagrange_at(tau, log_m)


@pytest.mark.parametrize("log_m", [1, 2, 3, 5])
def test_h_query_is_odd_half_of_double_basis(log_m):
    """H_query[j] = L_j(tau/g) Z(tau) / (-2 delta) = L^(2m)_(2j+1)(tau) / delta, g = omega_2m."""
    rng = random.Random(100 + log_m)
    tau, delta = rng.randrange(2, R), rng.randrange(1, R)
    m = 1 << log_m
    g = bn.root_of_unity(log_m + 1)
    zt = (pow(tau, m, R) - 1) % R
    h = [x * zt % R * pow(-2 * delta % R, -1, R) % R for x in g16.lagrange_at(tau, log_m, shift=g)]
    dinv = pow(delta, -1, R)
    assert h == [x * dinv % R for x in g16.lagrange_at(tau, log_m + 1)[1::2]]


def spec_ceremony(cs, log_max, seed):
    rng = random.Random(seed)
    acc = spec.ptau_to_bytes(spec.ptau_new(log_max))
    ts, as_, bs = [], [], []
    for _ in range(2):
        t, a, b = (rng.randrange(1, R) for _ in range(3))
        acc, _ = spec.contribute(acc, t, a, b, [rng.randrange(1, R) for _ in range(3)])
        ts.append(t); as_.append(a); bs.append(b)
    pk, vk = spec.prepare(acc, cs)
    ds = [rng.randrange(1, R) for _ in range(2)]
    for d in ds:
        pk, vk = spec.phase2_contribute(pk, vk, d)
    return pk, vk, (prod(ts), prod(as_), prod(bs), 1, prod(ds))


def test_spec_ceremony_key_equals_setup_with_the_products():
    cs = rand_circuit(random.Random(5), 1, 1, 3, unused=1)
    pk, vk, tw = spec_ceremony(cs, 3, 5)
    pk0, vk0 = g16.setup(cs, *tw)
    assert pk == pk0 and vk == vk0


def test_spec_verifier_rejects_tampering():
    rng = random.Random(7)
    acc0 = spec.ptau_to_bytes(spec.ptau_new(1))
    acc1, rec = spec.contribute(acc0, *(rng.randrange(1, R) for _ in range(3)), [rng.randrange(1, R) for _ in range(3)])
    assert spec.ptau_verify(acc0, acc1, rec)
    A = spec.ptau_from_bytes(acc1)
    bad_power = dict(A, tau1=A["tau1"][:2] + [bn.g1_add(A["tau1"][2], bn.G1_GEN)] + A["tau1"][3:])
    swapped = dict(A, alpha1=A["alpha1"][::-1])
    bad_z = rec[:-32] + ((int.from_bytes(rec[-32:], "little") + 1) % R).to_bytes(32, "little")
    assert not spec.ptau_verify(acc0, spec.ptau_to_bytes(bad_power), rec)
    assert not spec.ptau_verify(acc0, spec.ptau_to_bytes(swapped), rec)
    assert not spec.ptau_verify(acc0, acc1, bad_z)
    assert not spec.ptau_verify(acc1, acc1, rec)          # a record for another accumulator


def test_golden_matches_spec():
    g = json.load(open(GOLDEN))
    acc = spec.ptau_to_bytes(spec.ptau_new(g["log_max"]))
    assert acc.hex() == g["accumulators"][0]
    for c, nxt, rec in zip(g["contributors"], g["accumulators"][1:], g["records"]):
        acc, r = spec.contribute(acc, *c["secrets"], c["nonces"])
        assert acc.hex() == nxt and r.hex() == rec


# ---- GPU ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ctx():
    c = ob.Context(0)
    yield c
    c.close()


def scale(ctx, g2, pts, scalars, per_point):
    import ctypes as C
    n = len(pts) // (128 if g2 else 64)
    out = C.create_string_buffer(len(pts))
    api._check(api.lib().og_scale_points(ctx._h, g2, pts, scalars, n, per_point, out), ctx)
    return out.raw


def intt(ctx, g2, pts, log_m):
    import ctypes as C
    buf = C.create_string_buffer(bytes(pts), len(pts))
    api._check(api.lib().og_intt_points(ctx._h, g2, buf, log_m), ctx)
    return buf.raw


def gen_mul(ctx, g2, scalars):
    import ctypes as C
    out = C.create_string_buffer((128 if g2 else 64) * len(scalars))
    fn = api.lib().og_g2_generator_mul if g2 else api.lib().og_g1_generator_mul
    api._check(fn(ctx._h, b"".join(api.fr_bytes(x) for x in scalars), len(scalars), out), ctx)
    return out.raw


@pytest.mark.gpu
@pytest.mark.parametrize("g2", [0, 1])
def test_scale_points_edge_scalars(ctx, g2):
    rng = random.Random(11 + g2)
    ks = [0, 1, R - 1, 2, 1 << 64, 1 << 253, rng.randrange(R), rng.randrange(R)]
    base = [rng.randrange(1, R) for _ in ks]
    pts = bytearray(gen_mul(ctx, g2, base))
    PB = 128 if g2 else 64
    pts[PB:2 * PB] = bytes(PB)                          # a point at infinity
    mul, to_b, gen = (bn.g2_mul, bn.g2_to_bytes, bn.G2_GEN) if g2 else (bn.g1_mul, bn.g1_to_bytes, bn.G1_GEN)
    want = b"".join(to_b(None if i == 1 else mul(gen, b * k % R)) for i, (b, k) in enumerate(zip(base, ks)))
    assert scale(ctx, g2, bytes(pts), b"".join(api.fr_bytes(k) for k in ks), 1) == want
    assert scale(ctx, g2, bytes(pts), api.fr_bytes(R - 1), 0) == b"".join(
        to_b(None if i == 1 else mul(gen, -b % R)) for i, b in enumerate(base))


@pytest.mark.gpu
@pytest.mark.parametrize("g2,log_m", [(0, 3), (1, 3), (0, 12), (1, 12)])
def test_intt_of_powers_is_lagrange_basis(ctx, g2, log_m):
    tau = random.Random(log_m).randrange(2, R)
    m = 1 << log_m
    powers = gen_mul(ctx, g2, [pow(tau, i, R) for i in range(m)])
    assert intt(ctx, g2, powers, log_m) == gen_mul(ctx, g2, g16.lagrange_at(tau, log_m))


def contributors(rng, n):
    return [([rng.randrange(1, R) for _ in range(3)], [rng.randrange(1, R) for _ in range(3)]) for _ in range(n)]


@pytest.mark.gpu
def test_accumulator_bytes_match_golden_and_spec(ctx):
    g = json.load(open(GOLDEN))
    acc = ob.ptau_new(ctx, g["log_max"])
    assert acc.hex() == g["accumulators"][0]
    for c, nxt, rec in zip(g["contributors"], g["accumulators"][1:], g["records"]):
        acc2, r = ob.ptau_contribute(ctx, acc, c["secrets"], c["nonces"])
        assert acc2.hex() == nxt and r.hex() == rec
        assert ob.ptau_verify(ctx, acc, acc2, r)
        acc = acc2
    rng = random.Random(3)
    acc = ob.ptau_new(ctx, 4)
    sacc = spec.ptau_to_bytes(spec.ptau_new(4))
    for s, k in contributors(rng, 1):
        acc, r = ob.ptau_contribute(ctx, acc, s, k)
        sacc, sr = spec.contribute(sacc, *s, k)
        assert acc == sacc and r == sr


def ceremony(ctx, log_max, n, seed):
    """n contributors, each verified -> (accumulators, records, (prod t, prod a, prod b))"""
    rng = random.Random(seed)
    accs, recs, ps = [ob.ptau_new(ctx, log_max)], [], [1, 1, 1]
    for s, k in contributors(rng, n):
        acc, rec = ob.ptau_contribute(ctx, accs[-1], s, k)
        assert ob.ptau_verify(ctx, accs[-1], acc, rec)
        accs.append(acc); recs.append(rec)
        ps = [p * x % R for p, x in zip(ps, s)]
    return accs, recs, ps


@pytest.fixture(scope="module")
def acc8(ctx):
    """log_max 11: room for the deposit domain (2^10)"""
    return ceremony(ctx, 11, 3, 8)


def phase2(ctx, pk, vk, rng, n=2):
    d = 1
    for _ in range(n):
        x = rng.randrange(1, R)
        pk1, vk1, rec = ob.phase2_contribute(ctx, pk, vk, x, rng.randrange(1, R))
        assert ob.phase2_verify(ctx, pk, vk, pk1, vk1, rec)
        pk, vk, d = pk1, vk1, d * x % R
    return pk, vk, d


@pytest.mark.gpu
def test_three_contributors_verify(acc8):
    accs, recs, _ = acc8
    assert len(recs) == 3


@pytest.mark.gpu
def test_deposit_key_byte_identical_and_proves(ctx, acc8):
    accs, _, (t, a, b) = acc8
    pk, vk = ob.ptau_prepare_deposit(ctx, accs[-1])
    pk, vk, d = phase2(ctx, pk, vk, random.Random(1))
    assert (pk, vk) == ob.setup_deposit(ctx, t, a, b, 1, d)
    PK = ob.ProvingKey(ctx, pk)
    rng = random.Random(2)
    batch = 2
    nul, sec, dep = (b"".join(api.fr_bytes(rng.randrange(R)) for _ in range(batch)) for _ in range(3))
    rs = b"".join(api.fr_bytes(rng.randrange(R)) for _ in range(2 * batch))
    proofs, pub = PK.prove_deposit(nul, sec, dep, rs)
    assert all(ob.verify(vk, pub[64 * i:64 * i + 64], proofs[256 * i:256 * i + 256]) for i in range(batch))
    PK.close()


@pytest.mark.gpu
def test_transfer_key_byte_identical(ctx):
    accs, _, (t, a, b) = ceremony(ctx, 14, 1, 14)           # the depth-2 transfer domain is 2^14
    pk, vk = ob.ptau_prepare_transfer(ctx, accs[-1], 2)
    pk, vk, d = phase2(ctx, pk, vk, random.Random(3))
    assert (pk, vk) == ob.setup_transfer(ctx, 2, t, a, b, 1, d)
    PK = ob.ProvingKey(ctx, pk)
    assert PK.transfer_depth == 2
    PK.close()


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(0, 2, 5, 0, 0), (1, 3, 9, 2, 0), (2, 2, 7, 0, 2), (3, 4, 12, 1, 1), (1, 1, 6, 0, 0)])
def test_random_r1cs_keys_byte_identical(ctx, acc8, shape):
    n_pub, n_in, n_c, unused, empty = shape
    cs = rand_circuit(random.Random(sum(shape)), n_pub, n_in, n_c, unused=unused, empty_rows=empty)
    accs, _, (t, a, b) = acc8
    pk, vk = ob.ptau_prepare(ctx, accs[-1], cs.n_vars, cs.n_pub, cs.csr("A"), cs.csr("B"), cs.csr("C"))
    pk, vk, d = phase2(ctx, pk, vk, random.Random(9))
    assert (pk, vk) == ob.setup_r1cs(ctx, cs.n_vars, cs.n_pub, cs.csr("A"), cs.csr("B"), cs.csr("C"), t, a, b, 1, d)


@pytest.mark.gpu
def test_heavy_and_empty_columns(ctx, acc8):
    """ONE in every row of A and B (a column through the MSM engine) and a variable in no row (an empty column)."""
    from oracle.withdraw_circuit import R1CS
    nc, n_pub = 1000, 1
    cs = R1CS(3 + nc, n_pub)                    # ONE, x, an unused variable, one output per row
    for j in range(nc):
        cs.add({0: j + 1, 1: 1}, {0: 1}, {3 + j: 1})
    cs.add({1: 1}, {1: 1}, {3: 1})
    accs, _, (t, a, b) = ceremony(ctx, 10, 1, 4)
    pk, vk = ob.ptau_prepare(ctx, accs[-1], cs.n_vars, cs.n_pub, cs.csr("A"), cs.csr("B"), cs.csr("C"))
    assert (pk, vk) == ob.setup_r1cs(ctx, cs.n_vars, cs.n_pub, cs.csr("A"), cs.csr("B"), cs.csr("C"), t, a, b, 1, 1)


@pytest.mark.gpu
def test_withdraw32_key_byte_identical(ctx):
    accs, _, (t, a, b) = ceremony(ctx, 15, 1, 32)
    pk, vk = ob.ptau_prepare_withdraw(ctx, accs[-1], 32)
    pk, vk, d = phase2(ctx, pk, vk, random.Random(32), n=1)
    assert (pk, vk) == ob.setup_withdraw(ctx, 32, t, a, b, 1, d)
    PK = ob.ProvingKey(ctx, pk)
    assert PK.depth == 32
    PK.close()


def patch(blob, off, new):
    return blob[:off] + new + blob[off + len(new):]


@pytest.mark.gpu
def test_phase1_rejections(ctx):
    rng = random.Random(21)
    acc0 = ob.ptau_new(ctx, 3)
    (s, k), = contributors(rng, 1)
    acc1, rec = ob.ptau_contribute(ctx, acc0, s, k)
    assert ob.ptau_verify(ctx, acc0, acc1, rec)
    M = 8
    offs = {"tau1": 12, "alpha1": 12 + 128 * M, "beta1": 12 + 192 * M, "tau2": 12 + 256 * M}
    junk1, junk2 = gen_mul(ctx, 0, [12345]), gen_mul(ctx, 1, [12345])
    bad = [patch(acc1, offs[n] + 64 * 3, junk1) for n in ("tau1", "alpha1", "beta1")]
    bad.append(patch(acc1, offs["tau2"] + 128 * 3, junk2))
    bad.append(patch(acc1, 12 + 384 * M, junk2))                                  # beta_g2
    bad.append(patch(patch(acc1, 12 + 64 * 4, acc1[12 + 64 * 5:12 + 64 * 6]), 12 + 64 * 5, acc1[12 + 64 * 4:12 + 64 * 5]))
    off_curve = bytearray(acc1[12 + 64 * 2:12 + 64 * 3]); off_curve[32] ^= 1
    bad.append(patch(acc1, 12 + 64 * 2, bytes(off_curve)))
    bad.append(patch(acc1, offs["tau2"] + 128 * 2, twist_point_outside_subgroup()))
    for b in bad:
        assert not ob.ptau_verify(ctx, acc0, b, rec)
    z = int.from_bytes(rec[-32:], "little")
    assert not ob.ptau_verify(ctx, acc0, acc1, rec[:-32] + ((z + 1) % R).to_bytes(32, "little"))
    acc0b = ob.ptau_contribute(ctx, acc0, [2, 3, 4], [5, 6, 7])[0]
    assert not ob.ptau_verify(ctx, acc0b, acc1, rec)                              # a record for another accumulator


def twist_point_outside_subgroup():
    """A point of the twist E'(Fq2) found by try-and-increment on x, without cofactor clearing (so not in G2)."""
    P = bn.P
    def f2_sqrt(a):
        # Fq2 square root (p = 3 mod 4): the standard complex method
        a0, a1 = a
        if a1 == 0:
            r = pow(a0, (P + 1) // 4, P)
            if r * r % P == a0:
                return (r, 0)
            r = pow(-a0 % P, (P + 1) // 4, P)
            return (0, r) if r * r % P == -a0 % P else None
        n = (a0 * a0 + a1 * a1) % P
        s = pow(n, (P + 1) // 4, P)
        if s * s % P != n:
            return None
        for t in ((a0 + s) * pow(2, -1, P) % P, (a0 - s) * pow(2, -1, P) % P):
            x0 = pow(t, (P + 1) // 4, P)
            if x0 * x0 % P == t and x0:
                return (x0, a1 * pow(2 * x0, -1, P) % P)
        return None
    x = 1
    while True:
        xx = (x, 1)
        rhs = bn.f2_add(bn.f2_mul(bn.f2_mul(xx, xx), xx), bn.G2_B)
        y = f2_sqrt(rhs)
        if y is not None and bn.f2_mul(y, y) == rhs:
            pt = (xx, y)
            assert bn.g2_on_curve(pt) and bn.g2_add(bn.g2_mul(pt, R - 1), pt) is not None     # r P != infinity
            return bn.g2_to_bytes(pt)
        x += 1


@pytest.mark.gpu
def test_phase2_rejections(ctx, acc8):
    accs, _, _ = acc8
    pk, vk = ob.ptau_prepare_deposit(ctx, accs[-1])
    rng = random.Random(5)
    pk1, vk1, rec = ob.phase2_contribute(ctx, pk, vk, rng.randrange(1, R), rng.randrange(1, R))
    assert ob.phase2_verify(ctx, pk, vk, pk1, vk1, rec)
    qa = 28 + 64 + 64 + 128 + 64 + 128
    assert not ob.phase2_verify(ctx, pk, vk, patch(pk1, qa + 64, gen_mul(ctx, 0, [7])), vk1, rec)
    # an L point scaled by the wrong d
    info = ob.deposit_r1cs_info()
    nv = info["n_vars"]
    ql = qa + 64 * nv * 2 + 128 * nv
    wrong = scale(ctx, 0, pk[ql:ql + 64], api.fr_bytes(3), 0)
    assert not ob.phase2_verify(ctx, pk, vk, patch(pk1, ql, wrong), vk1, rec)
    z = int.from_bytes(rec[-32:], "little")
    assert not ob.phase2_verify(ctx, pk, vk, pk1, vk1, rec[:-32] + ((z + 1) % R).to_bytes(32, "little"))


@pytest.mark.gpu
def test_invalid_arguments(ctx):
    with pytest.raises(ob.OwshenB200Error) as e:
        ob.ptau_new(ctx, 0)
    assert e.value.code == api.OG_E_INVALID
    with pytest.raises(ob.OwshenB200Error):
        ob.ptau_new(ctx, 25)
    acc = ob.ptau_new(ctx, 2)
    for bad in (b"XGPT" + acc[4:], acc[:-1]):
        with pytest.raises(ob.OwshenB200Error) as e:
            ob.ptau_contribute(ctx, bad, [1, 2, 3], [1, 2, 3])
        assert e.value.code == api.OG_E_INVALID
    with pytest.raises(ob.OwshenB200Error) as e:
        ob.ptau_contribute(ctx, acc, [1, 0, 3], [1, 2, 3])
    assert e.value.code == api.OG_E_INVALID
    with pytest.raises(ob.OwshenB200Error) as e:
        ob.ptau_prepare_deposit(ctx, acc)                  # the deposit domain is larger than M = 4
    assert e.value.code == api.OG_E_INVALID
