"""og_groth16_setup: the development setup of any R1CS.  Keys and proofs of random small circuits against the oracle's
(cport.setup_bytes, cport.Prover), and every malformed input refused with its error code before any work starts."""
import ctypes as C
import random

import pytest

import owshen_b200 as ob
from owshen_b200 import api
from oracle import bn254 as bn
from oracle import cport
from oracle import groth16 as g16
from oracle.withdraw_circuit import R1CS, lc_eval
from tests.helpers import pk_blob, vk_blob

R = bn.R
OG_E_INVALID, OG_E_ENCODING = -1, -2


def rand_lc(rng, n_assigned, n_terms):
    """n_terms distinct variables among the first n_assigned, random non-zero coefficients (some small, some near r)."""
    vs = rng.sample(range(n_assigned), min(n_terms, n_assigned))
    return {v: rng.choice([1, 2, R - 1, rng.randrange(1, R)]) for v in vs}


def rand_circuit(rng, n_pub, n_inputs, n_constraints, max_terms=4, unused=0, empty_rows=0):
    """A satisfiable R1CS and witnesses for it.  Variables: ONE, n_pub public, n_inputs free private inputs, then one
    output per constraint (C = that output, so (A.w)(B.w) = out), then `unused` variables that appear in no constraint.
    The public inputs are bound by one constraint each, x * x = out.  `empty_rows` constraints have an empty A or B (C empty)."""
    n_vars = 1 + n_pub + n_inputs + n_constraints + unused
    cs = R1CS(n_vars, n_pub)
    first_out = 1 + n_pub + n_inputs
    for j in range(n_constraints):
        out = first_out + j
        if j < n_pub:
            a = b = {1 + j: 1}
        else:
            a = rand_lc(rng, out, rng.randrange(1, max_terms + 1))
            b = rand_lc(rng, out, rng.randrange(1, max_terms + 1))
        if j >= n_constraints - empty_rows:
            (a, b) = ({}, b) if j % 2 else (a, {})
            cs.add(a, b, {})
        else:
            cs.add(a, b, {out: 1})
    return cs


def rand_witness(rng, cs):
    w = [1] + [rng.randrange(R) for _ in range(cs.n_vars - 1)]
    for a, b, c in zip(cs.A, cs.B, cs.C):
        if c:
            (out,) = c
            w[out] = lc_eval(a, w) * lc_eval(b, w) % R
    assert cs.is_satisfied(w)
    return w


def lib_setup(ctx, cs, tw):
    return ob.setup_r1cs(ctx, cs.n_vars, cs.n_pub, cs.csr("A"), cs.csr("B"), cs.csr("C"), *tw)


# ---- CPU: argument checks at the Python boundary ------------------------------------------------------------------------
def test_setup_r1cs_checks_lengths():
    cs = rand_circuit(random.Random(1), 1, 2, 5)
    A, B, Cm = cs.csr("A"), cs.csr("B"), cs.csr("C")
    tw = [2, 3, 4, 5, 6]
    bad = [
        (A[:2], B, Cm),                                    # not a triple
        (A, (B[0][:-1], B[1], B[2]), Cm),                  # row_ptr of another length than A's
        (A, B, (Cm[0], Cm[1] + [1], Cm[2])),               # col_idx and coeffs differ
        ((A[0][:-1] + [A[0][-1] + 1], A[1], A[2]), B, Cm),  # row_ptr ends past the terms
        (([0], [], []), ([0], [], []), ([0], [], [])),     # no constraint
        (A, B, (Cm[0], [x - 2 ** 32 for x in Cm[1]], Cm[2])),   # negative column
    ]
    for mats in bad:
        with pytest.raises(ValueError):
            ob.setup_r1cs(None, cs.n_vars, cs.n_pub, *mats, *tw)


def test_random_circuits_are_satisfiable():
    rng = random.Random(2)
    for n_pub in (0, 1, 3):
        cs = rand_circuit(rng, n_pub, 3, 12, unused=2, empty_rows=2)
        rand_witness(rng, cs)


# ---- GPU ------------------------------------------------------------------------------------------------------------------
CASES = {
    # name: (n_pub, n_inputs, n_constraints, max_terms, unused, empty_rows)
    "no-public-inputs": (0, 3, 20, 3, 0, 0),
    "unused-variables": (2, 4, 30, 3, 3, 0),
    "empty-a-or-b-rows": (1, 2, 25, 3, 0, 4),
    "dozens-of-terms": (3, 5, 40, 48, 0, 0),
    "domain-exactly-full": (3, 2, 60, 4, 1, 2),      # 60 + 3 + 1 = 64 = 2^6
    "one-constraint": (0, 1, 1, 1, 0, 0),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_generic_setup_and_proofs_match_oracle(ctx, name):
    n_pub, n_inputs, n_constraints, max_terms, unused, empty_rows = CASES[name]
    rng = random.Random(name)
    cs = rand_circuit(rng, n_pub, n_inputs, n_constraints, max_terms, unused, empty_rows)
    if name == "domain-exactly-full":
        assert cs.n_constraints + cs.n_pub + 1 == 1 << g16.domain_log(cs.n_constraints, cs.n_pub)
    tw = [rng.randrange(1, R) for _ in range(5)]
    pk, vk = lib_setup(ctx, cs, tw)
    pkb, vkb = cport.setup_bytes(cs, *tw)
    assert pk == pk_blob(cs, pkb, 0)
    assert vk == vk_blob(vkb, n_pub)
    if unused:
        # a variable in no constraint has u = v = w = 0: its A, B1, B2 and L queries are the point at infinity
        i = cs.n_vars - 1
        assert pkb["a"][64 * i:64 * i + 64] == bytes(64) and pkb["l"][64 * (i - n_pub - 1):64 * (i - n_pub)] == bytes(64)
    batch = 5
    wits = [rand_witness(rng, cs) for _ in range(batch)]
    wbytes = b"".join(cport.frs(w) for w in wits)
    rs = cport.frs([rng.randrange(R) for _ in range(2 * batch)])
    PK = ob.ProvingKey(ctx, pk)
    try:
        assert (PK.n_vars, PK.n_pub, PK.depth) == (cs.n_vars, n_pub, 0)
        proofs = PK.prove_witnesses(wbytes, rs)
    finally:
        PK.close()
    assert proofs == cport.Prover(cs, pkb).prove_batch(wbytes, rs)
    for i, w in enumerate(wits):
        pub = cport.frs(w[1:n_pub + 1])
        assert ob.verify(vk, pub, proofs[256 * i:256 * i + 256]), i
        if n_pub:
            bad = bytearray(pub); bad[0] ^= 1
            assert not ob.verify(vk, bytes(bad), proofs[256 * i:256 * i + 256]), i


def _raw_setup(ctx, n_constraints, n_vars, n_pub, mats, toxic=None, full=False):
    """og_groth16_setup straight through ctypes (past the Python checks): the size query, or the whole setup."""
    args = []
    for ptr, col, val in mats:
        # an int row_ptr stands for that many zeros (empty rows), made without a Python list
        ptr = (C.c_uint32 * ptr)() if isinstance(ptr, int) else (C.c_uint32 * max(1, len(ptr)))(*ptr)
        args += [ptr, (C.c_uint32 * max(1, len(col)))(*col), val if isinstance(val, bytes) else cport.frs(val)]
    toxic = toxic or cport.frs([5, 6, 7, 8, 9])
    pl, vl = C.c_uint64(), C.c_uint64()
    rc = api.lib().og_groth16_setup(ctx._h, n_constraints, n_vars, n_pub, *args, toxic, None, C.byref(pl), None, C.byref(vl))
    if rc != 0 or not full:
        return rc
    pk, vk = C.create_string_buffer(pl.value), C.create_string_buffer(vl.value)
    return api.lib().og_groth16_setup(ctx._h, n_constraints, n_vars, n_pub, *args, toxic, pk, C.byref(pl), vk, C.byref(vl))


@pytest.mark.gpu
def test_generic_setup_rejects_malformed_input(ctx):
    rng = random.Random(7)
    cs = rand_circuit(rng, 2, 3, 10)
    nc, nv, npub = cs.n_constraints, cs.n_vars, cs.n_pub
    good = [cs.csr(m) for m in "ABC"]
    assert _raw_setup(ctx, nc, nv, npub, good, full=True) == 0

    def with_matrix(k, ptr=None, col=None, val=None):
        mats = list(good)
        p, c, v = mats[k]
        mats[k] = (ptr if ptr is not None else p, col if col is not None else c, val if val is not None else v)
        return mats

    for k in range(3):
        p, c, v = good[k]
        assert _raw_setup(ctx, nc, nv, npub, with_matrix(k, ptr=[1] + p[1:])) == OG_E_INVALID, k           # row_ptr[0] != 0
        dec = list(p); dec[1] = p[-1] + 1                 # ends at nnz, but row 1 starts past row 2
        assert _raw_setup(ctx, nc, nv, npub, with_matrix(k, ptr=dec)) == OG_E_INVALID, k                  # row_ptr decreases
        col = list(c); col[-1] = nv
        assert _raw_setup(ctx, nc, nv, npub, with_matrix(k, col=col)) == OG_E_INVALID, k                  # column >= n_vars
        col[-1] = 0xFFFFFFFF
        assert _raw_setup(ctx, nc, nv, npub, with_matrix(k, col=col)) == OG_E_INVALID, k
        val = cport.frs(v[:-1]) + R.to_bytes(32, "little")
        assert _raw_setup(ctx, nc, nv, npub, with_matrix(k, val=val)) == OG_E_ENCODING, k                 # coefficient >= r
        val = cport.frs(v[:-1]) + b"\xff" * 32
        assert _raw_setup(ctx, nc, nv, npub, with_matrix(k, val=val)) == OG_E_ENCODING, k
    empty = [([0], [], [])] * 3
    assert _raw_setup(ctx, 0, nv, npub, empty) == OG_E_INVALID                                          # no constraint
    assert _raw_setup(ctx, nc, npub, npub, good) == OG_E_INVALID                                        # n_pub + 1 > n_vars
    assert _raw_setup(ctx, nc, 0, 0, good) == OG_E_INVALID
    big = 1 << 16
    rows = [(nc + 1, [], [])] * 3
    assert _raw_setup(ctx, nc, big + 2, big + 1, rows) == OG_E_INVALID                                  # n_pub > 2^16
    assert _raw_setup(ctx, nc, big + 1, big, rows) == 0                                                 # n_pub = 2^16 is allowed
    n_max = (1 << 24) - npub - 1                                                                         # domain exactly 2^24
    assert _raw_setup(ctx, n_max + 1, nv, npub, [(n_max + 2, [], [])] * 3) == OG_E_INVALID               # domain above 2^24
    assert _raw_setup(ctx, n_max, nv, npub, [(n_max + 1, [], [])] * 3) == 0                              # size query at 2^24
    # toxic values that put tau or tau / g in the domain
    log_m = g16.domain_log(nc, npub)
    g = bn.root_of_unity(log_m + 1)
    w = bn.root_of_unity(log_m)
    for tau in (1, w, g, g * w % R):
        assert _raw_setup(ctx, nc, nv, npub, good, toxic=cport.frs([tau, 6, 7, 8, 9]), full=True) == OG_E_INVALID, tau
    assert _raw_setup(ctx, nc, nv, npub, good, toxic=cport.frs([5, 6, 7, 0, 9]), full=True) == OG_E_INVALID        # gamma = 0
    assert _raw_setup(ctx, nc, nv, npub, good, toxic=R.to_bytes(32, "little") + cport.frs([6, 7, 8, 9]), full=True) == OG_E_ENCODING
    # the context is still usable: a valid setup right after matches the oracle
    tw = [rng.randrange(1, R) for _ in range(5)]
    pk, vk = lib_setup(ctx, cs, tw)
    pkb, vkb = cport.setup_bytes(cs, *tw)
    assert pk == pk_blob(cs, pkb, 0) and vk == vk_blob(vkb, npub)
    with pytest.raises(ob.OwshenB200Error) as e:
        lib_setup(ctx, cs, [1, 2, 3, 4, 5])
    assert e.value.code == OG_E_INVALID
