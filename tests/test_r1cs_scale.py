"""The generic R1CS prover (og_groth16_setup, og_groth16_prove, og_groth16_h_evals) at real circuit sizes and degenerate key
shapes, and og_ntt at every pass plan, against the oracle's C port.

ntt_mont_dev plans one pass for log_n <= 10, two for 11..17, three for 18..24 and four for 25..27; the prover runs its
folded pair (an inverse transform without 1/n, then a forward coset transform whose factors carry it) at the key's log_m.
Circuits here are CSR arrays built with numpy (CsrCircuit), not the dict-based R1CS of the smaller tests, and the
oracle's key is read back from the library's key blob (parse_pk) except where cport.setup_bytes checks that blob."""
import contextlib
import ctypes as C
import operator
import random
import struct

import numpy as np
import pytest

import owshen_b200 as ob
from owshen_b200 import api
from oracle import bn254 as bn
from oracle import cport
from oracle import groth16 as g16
from oracle.withdraw_circuit import R1CS
from tests.helpers import pk_blob, vk_blob

R = bn.R
GIB = 1 << 30
LANE_BUDGET = 28 << 30            # groth16.cu: LANE_SCRATCH_BUDGET
GRID_Y_MAX = 65535                # the prover's NTT puts 3 transforms per proof of a chunk on grid.y
NTT_MODES = [(False, False), (True, False), (False, True), (True, True)]       # (inverse, coset)

# coefficients: a palette of base values times a palette of row scales, so that coefficient bytes are one table lookup
_crng = random.Random(1729)
PALETTE = [1, 2, 3, R - 1, R - 2] + [_crng.randrange(R) for _ in range(11)]
SCALES = [1, 2, R - 1] + [_crng.randrange(1, R) for _ in range(13)]
COEF = [p * s % R for p in PALETTE for s in SCALES]                  # code p * 16 + q
COEF_BYTES = np.frombuffer(cport.frs(COEF), dtype=np.uint8).reshape(-1, 32)
EDGES = (0, 1, R - 1)


@contextlib.contextmanager
def own_context():
    """A context of its own: its scratch and NTT tables are released when the test ends, not kept by the session's."""
    c = ob.Context(0)
    try:
        yield c
    finally:
        c.close()


# ---- circuits as CSR arrays -------------------------------------------------------------------------------------------
class CsrCircuit:
    """A satisfiable R1CS as CSR arrays.  Variables: ONE, n_in inputs, then n_out outputs; the first n_pub after ONE are
    public.  Output t is LA_t(w) * LB_t(w) for linear combinations of ONE and the inputs; constraint j proves output
    t = j mod n_out as (s_j LA_t) * LB_t = s_j out_t, so a domain can be large while the variables stay few.  With
    `empty_b` there are no outputs and B and C are empty: every row is s_j LA_t * 0 = 0."""

    def __init__(self, seed, n_pub, n_in, n_out, n_constraints, max_terms=3, empty_b=False, one_in_every_row=False,
                 heavy=0, duplicate=False):
        assert not (empty_b and n_out)
        rng = random.Random(seed)
        self.n_in, self.n_out, self.n_pub = n_in, n_out, n_pub
        self.n_vars = 1 + n_in + n_out
        self.n_constraints = n_constraints
        assert n_pub + 1 <= self.n_vars
        n_base = n_out if n_out else min(n_constraints, 1024)

        def lc(t):
            k = heavy if (t == 0 and heavy) else rng.randrange(1, max_terms + 1)
            cols = rng.sample(range(1 + n_in), min(k, 1 + n_in))
            if one_in_every_row and 0 not in cols:
                cols[0] = 0
            if t == 0 and duplicate:
                cols = cols + [cols[0]]              # the same variable twice in one row, with its own coefficient
            return [(v, rng.randrange(16)) for v in cols]

        self.la = [lc(t) for t in range(n_base)]
        self.lb = [] if empty_b else [lc(t) for t in range(n_base)]
        t_row = np.arange(n_constraints, dtype=np.int64) % n_base
        q_row = np.array([0 if j < n_base else rng.randrange(16) for j in range(n_constraints)], dtype=np.int64)
        self.mats = {"A": self._rows(self.la, t_row, q_row), "B": self._rows(self.lb, t_row, None)}
        if n_out:
            ptr = np.arange(n_constraints + 1, dtype=np.uint32)
            self.mats["C"] = (ptr, (1 + n_in + t_row).astype(np.uint32), q_row)          # PALETTE[0] = 1: code q = SCALES[q]
        else:
            self.mats["C"] = self._rows([], t_row, None)
        self._csr = {}

    def _rows(self, base, t_row, q_row):
        """CSR of rows j = base[t_row[j]] scaled by SCALES[q_row[j]] (no scale when q_row is None)."""
        n = len(t_row)
        if not base:
            return np.zeros(n + 1, dtype=np.uint32), np.zeros(0, dtype=np.uint32), np.zeros(0, dtype=np.int64)
        cnt = np.array([len(x) for x in base], dtype=np.int64)
        bptr = np.concatenate([[0], np.cumsum(cnt)])
        bcol = np.array([v for x in base for v, _ in x], dtype=np.uint32)
        bcode = np.array([p for x in base for _, p in x], dtype=np.int64) * 16
        counts = cnt[t_row]
        ptr = np.concatenate([[0], np.cumsum(counts)])
        idx = np.repeat(bptr[t_row], counts) + (np.arange(ptr[-1]) - np.repeat(ptr[:-1], counts))
        code = bcode[idx] if q_row is None else bcode[idx] + np.repeat(q_row, counts)
        return ptr.astype(np.uint32), bcol[idx], code

    def raw(self, which):
        """(row_ptr, col_idx, coefficient bytes) as og_groth16_setup takes them."""
        ptr, col, code = self.mats[which]
        return ptr, col, COEF_BYTES[code].tobytes()

    def csr(self, which):
        """(row_ptr, col_idx, coeffs) as lists, as R1CS.csr gives them (what cport.Prover and pk_blob read)."""
        if which not in self._csr:
            ptr, col, code = self.mats[which]
            self._csr[which] = (ptr.tolist(), col.tolist(), [COEF[c] for c in code.tolist()])
        return self._csr[which]

    def as_r1cs(self):
        """The dict-based R1CS of the same rows (for cport.setup_bytes; needs no duplicate variable in a row)."""
        cs = R1CS(self.n_vars, self.n_pub)
        mats = [self.csr(m) for m in "ABC"]
        for j in range(self.n_constraints):
            rows = [dict(zip(col[ptr[j]:ptr[j + 1]], val[ptr[j]:ptr[j + 1]])) for ptr, col, val in mats]
            assert all(len(r) == ptr[j + 1] - ptr[j] for r, (ptr, _, _) in zip(rows, mats))
            cs.add(*rows)
        return cs

    def witness(self, rng, pub_below=R):
        """A satisfying assignment: random inputs (some 0, 1 and r - 1), outputs from them.  Public inputs below
        `pub_below` keep the host verifier's scalar multiplications short when there are 2^16 of them."""
        w = [1] + [rng.randrange(pub_below) if i < self.n_pub and pub_below < R else
                   rng.choice(EDGES) if i % 7 == 3 else rng.randrange(R) for i in range(self.n_in)]
        ev = lambda terms: sum(COEF[p * 16] * w[v] for v, p in terms)
        return w + [ev(a) * ev(b) % R for a, b in zip(self.la[:self.n_out], self.lb)]

    def random_witness(self, rng, edges_only=False):
        """Any assignment (h_evals sets c = a * b on the domain, so it need not satisfy the circuit)."""
        if edges_only:
            return [1] + [rng.choice(EDGES) for _ in range(self.n_vars - 1)]
        return [1] + [rng.choice(EDGES) if i % 5 == 0 else rng.randrange(R) for i in range(self.n_vars - 1)]

    def is_satisfied(self, w):
        for j in range(self.n_constraints):
            a, b, c = (sum(val[k] * w[col[k]] for k in range(ptr[j], ptr[j + 1])) % R for ptr, col, val in (self.csr(m) for m in "ABC"))
            if a * b % R != c:
                return False
        return True


def domain_circuit(seed, log_m, fill, n_pub=3, **kw):
    """A circuit whose domain is 2^log_m: exactly full (n_constraints + n_pub + 1 = 2^log_m) or just over half full."""
    need = (1 << log_m) if fill == "full" else (1 << (log_m - 1)) + 1
    n_pub = max(0, min(n_pub, need - 2))
    nc = need - n_pub - 1
    kw.setdefault("n_out", max(1, min(nc, 2048)))
    cs = CsrCircuit(seed, n_pub, kw.pop("n_in", 64), n_constraints=nc, **kw)
    assert g16.domain_log(cs.n_constraints, cs.n_pub) == log_m
    return cs


def gpu_setup(ctx, cs, tw):
    """og_groth16_setup on the circuit's arrays (no Python lists at large sizes) -> (pk, vk)."""
    keep, args = [], []
    for m in "ABC":
        ptr, col, val = cs.raw(m)
        col = col if len(col) else np.zeros(1, dtype=np.uint32)
        keep += [ptr, col, val]
        args += [ptr.ctypes.data, col.ctypes.data, val]
    toxic = cport.frs(tw)
    pl, vl = C.c_uint64(), C.c_uint64()
    setup = api.lib().og_groth16_setup
    api._check(setup(ctx._h, cs.n_constraints, cs.n_vars, cs.n_pub, *args, toxic, None, C.byref(pl), None, C.byref(vl)), ctx)
    pk, vk = C.create_string_buffer(pl.value), C.create_string_buffer(vl.value)
    api._check(setup(ctx._h, cs.n_constraints, cs.n_vars, cs.n_pub, *args, toxic, pk, C.byref(pl), vk, C.byref(vl)), ctx)
    return pk.raw[:pl.value], vk.raw[:vl.value]


def parse_pk(blob):
    """The inverse of tests.helpers.pk_blob: (header, the oracle's pk dict, [(row_ptr, col, coefficient bytes) of A, B])."""
    magic, version, depth, nc, nv, n_pub, log_m = struct.unpack_from("<4s6I", blob)
    assert (magic, version) == (b"OGPK", 1)
    off = 28

    def take(n):
        nonlocal off
        off += n
        assert off <= len(blob)
        return blob[off - n:off]

    pkb = dict(log_m=log_m, n_vars=nv, n_pub=n_pub)
    for name, size in (("alpha1", 64), ("beta1", 64), ("beta2", 128), ("delta1", 64), ("delta2", 128), ("a", 64 * nv),
                       ("b1", 64 * nv), ("b2", 128 * nv), ("l", 64 * (nv - n_pub - 1)), ("h", 64 << log_m)):
        pkb[name] = take(size)
    csr = []
    for _ in "AB":
        (nnz,) = struct.unpack("<I", take(4))
        csr.append((np.frombuffer(take(4 * (nc + 1)), dtype="<u4"), np.frombuffer(take(4 * nnz), dtype="<u4"), take(32 * nnz)))
    assert off == len(blob)
    return dict(depth=depth, n_constraints=nc, n_vars=nv, n_pub=n_pub, log_m=log_m), pkb, csr


def key_and_oracle(ctx, cs, tw):
    """The library's key for cs, checked to hold the circuit's shape and A, B, and the oracle's pk dict read from it."""
    pk, vk = gpu_setup(ctx, cs, tw)
    hdr, pkb, csr = parse_pk(pk)
    assert hdr == dict(depth=0, n_constraints=cs.n_constraints, n_vars=cs.n_vars, n_pub=cs.n_pub,
                       log_m=g16.domain_log(cs.n_constraints, cs.n_pub))
    for (ptr, col, val), m in zip(csr, "AB"):
        p, c, v = cs.raw(m)
        assert np.array_equal(ptr, p) and np.array_equal(col, c) and val == v, m
    return pk, vk, pkb


def check_proofs(vk, cs, wits, proofs):
    """Every proof verifies with its public inputs, and not with the first of them changed."""
    for i, w in enumerate(wits):
        pub, proof = cport.frs(w[1:cs.n_pub + 1]), proofs[256 * i:256 * i + 256]
        assert ob.verify(vk, pub, proof), i
        if cs.n_pub:
            assert not ob.verify(vk, cport.frs([(w[1] + 1) % R]) + pub[32:], proof), i


def rand_rs(rng, n):
    return cport.frs([rng.randrange(R) for _ in range(2 * n)])


# ---- CPU: the circuits the GPU tests build --------------------------------------------------------------------------------
def test_csr_circuits_are_satisfiable_and_shaped():
    rng = random.Random(3)
    shapes = [dict(n_pub=2, n_in=5, n_out=7, n_constraints=40), dict(n_pub=3, n_in=40, n_out=6, n_constraints=30, heavy=35),
              dict(n_pub=1, n_in=4, n_out=5, n_constraints=20, duplicate=True, one_in_every_row=True),
              dict(n_pub=9, n_in=4, n_out=5, n_constraints=12), dict(n_pub=0, n_in=6, n_out=0, n_constraints=9, empty_b=True)]
    for i, kw in enumerate(shapes):
        cs = CsrCircuit(i, **kw)
        w = cs.witness(rng)
        assert len(w) == cs.n_vars and cs.is_satisfied(w), kw
        bad = list(w); bad[-1] = (bad[-1] + 1) % R
        assert kw.get("empty_b") or not cs.is_satisfied(bad), kw
        ptr, col, val = cs.raw("A")
        assert len(ptr) == cs.n_constraints + 1 and ptr[-1] == len(col) == len(val) // 32
        assert cport.frs(cs.csr("A")[2]) == val
    cs = CsrCircuit(0, **shapes[2])
    ptr, col, _ = cs.csr("A")
    assert len(set(col[ptr[0]:ptr[1]])) == ptr[1] - ptr[0] - 1                      # row 0 names one variable twice
    assert all(0 in col[ptr[j]:ptr[j + 1]] for j in range(cs.n_constraints))       # ONE in every row
    assert CsrCircuit(1, **shapes[1]).csr("B")[0][1] == 35                          # a heavy row
    cs = CsrCircuit(4, **shapes[4])
    assert cs.csr("B")[0] == cs.csr("C")[0] == [0] * (cs.n_constraints + 1)
    for log_m in (1, 2, 5):
        for fill in ("full", "half"):
            domain_circuit(log_m, log_m, fill)


def test_parse_pk_inverts_pk_blob():
    """parse_pk reads back what pk_blob writes, from an oracle key of a small circuit."""
    cs = CsrCircuit(5, 2, 3, 4, 9)
    pkb, _ = cport.setup_bytes(cs.as_r1cs(), 2, 3, 4, 5, 6)
    hdr, back, csr = parse_pk(pk_blob(cs, pkb, 7))
    assert hdr == dict(depth=7, n_constraints=9, n_vars=cs.n_vars, n_pub=2, log_m=4)
    assert all(back[k] == pkb[k] for k in pkb)
    assert [(list(p), list(c), v) for p, c, v in csr] == [(cs.csr(m)[0], cs.csr(m)[1], cport.frs(cs.csr(m)[2])) for m in "AB"]


# ---- A. og_ntt at every plan shape ----------------------------------------------------------------------------------------
def fr_array(nrng, n):
    """n values below 2^253 < r as an (n, 4) array of little-endian uint64 limbs, with 0, 1 and r - 1 at the ends."""
    a = np.frombuffer(nrng.bytes(32 * n), dtype=np.uint64).reshape(n, 4).copy()
    a[:, 3] &= np.uint64((1 << 61) - 1)
    edges = np.frombuffer(cport.frs([0, 1, R - 1]), dtype=np.uint64).reshape(3, 4)
    a[:3] = edges
    a[-3:] = edges
    return a


@pytest.mark.gpu
@pytest.mark.parametrize("log_n,batch", [(18, 2), (19, 1), (20, 1), (21, 1), (22, 1), (25, 1)])
def test_ntt_matches_oracle_at_three_and_four_passes(log_n, batch):
    """Full transforms in all four modes against cport.ntt: three passes at 2^18..2^22 (the later passes' K = 4, 5/4,
    5/5, 6/5, 6/6 cover both parities), four at 2^25; two transforms at 2^18 put grid.y = 2 over the in-place middle pass."""
    n = 1 << log_n
    data = fr_array(np.random.default_rng(log_n), batch * n).tobytes()
    with own_context() as c:
        for inverse, coset in NTT_MODES:
            got = c.ntt(data, log_n, batch, inverse, coset)
            for b in range(batch):
                row = slice(32 * n * b, 32 * n * (b + 1))
                assert got[row] == cport.ntt(data[row], inverse, coset), (inverse, coset, b)


def sparse_transform_at(pos, vals, log_n, ks):
    """{mode: [out[k] for k in ks]} of the four transforms of the vector with vals at pos and zeros elsewhere, exactly:
    forward sum x_j w^(jk), coset sum x_j g^j w^(jk), inverse n^-1 sum x_j w^(-jk), inverse coset that times g^(-k).
    ks is made of runs of consecutive indices, so each run steps every term w^(jk) by one product."""
    n = 1 << log_n
    w, g = bn.root_of_unity(log_n), bn.root_of_unity(log_n + 1)
    n_inv, g_inv = pow(n, -1, R), pow(g, -1, R)
    xc = [x * pow(g, p, R) % R for x, p in zip(vals, pos)]
    runs, start = [], 0
    for i in range(1, len(ks) + 1):
        if i == len(ks) or ks[i] != ks[i - 1] + 1:
            runs.append((ks[start], i - start))
            start = i
    out = {mode: [] for mode in NTT_MODES}
    dot = lambda a, b: sum(map(operator.mul, a, b)) % R
    for k0, length in runs:
        for base in (w, pow(w, -1, R)):
            step = [pow(base, p, R) for p in pos]
            cur = [pow(base, p * k0 % n, R) for p in pos]
            for k in range(k0, k0 + length):
                if base == w:
                    out[(False, False)].append(dot(vals, cur))
                    out[(False, True)].append(dot(xc, cur))
                else:
                    s = dot(vals, cur) * n_inv % R
                    out[(True, False)].append(s)
                    out[(True, True)].append(s * pow(g_inv, k, R) % R)
                cur = list(map(lambda a, b: a * b % R, cur, step))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("log_n", [26, 27])
def test_ntt_four_passes_on_sparse_input(log_n):
    """2^26 and 2^27 (the API's largest): 1000 random nonzero entries, 4096 outputs in 64 runs of 64 checked against the
    exact sums.  After the first stages every butterfly carries dense data, so the whole four-pass plan is exercised; a
    round trip would not catch a consistently wrong root of unity, these sums do."""
    n = 1 << log_n
    rng = random.Random(log_n)
    pos = sorted(rng.sample(range(n), 1000))
    vals = [rng.randrange(R) for _ in pos]
    vals[:3] = EDGES[::-1]
    starts = sorted({0, n - 64} | {rng.randrange(64, n - 128) & ~63 for _ in range(62)})
    while len(starts) < 64:
        starts = sorted(set(starts) | {rng.randrange(64, n - 128) & ~63})
    ks = [s + i for s in starts for i in range(64)]
    want = sparse_transform_at(pos, vals, log_n, ks)
    limbs = np.frombuffer(cport.frs(vals), dtype=np.uint64).reshape(-1, 4)
    arr = np.zeros((n, 4), dtype=np.uint64)
    with own_context() as c:
        for inverse, coset in NTT_MODES:
            arr[:] = 0
            arr[pos] = limbs
            api._check(api.lib().og_ntt(c._h, arr.ctypes.data, log_n, 1, int(inverse), int(coset)), c)
            got = cport.unfr(arr[ks].tobytes())
            bad = [k for k, x, y in zip(ks, got, want[(inverse, coset)]) if x != y]
            assert not bad, (inverse, coset, len(bad), bad[:8])


# ---- B. the folded transform pair through og_groth16_h_evals --------------------------------------------------------------
H_LOGS = [1, 2, 3, 5, 9, 10, 11, 12, 13, 16, 17, 18, 19, 20, 21]


@pytest.mark.gpu
@pytest.mark.parametrize("log_m", H_LOGS)
def test_h_evals_match_oracle_at_every_plan_shape(ctx, log_m):
    """PK.h_evals against the oracle's h_evals byte for byte, at every pass plan the prover reaches below 2^22 (one pass
    up to 2^10, two up to 2^17, three above), for a domain exactly full and one just over half full; random witnesses
    (c = a * b on the domain on both sides, so they need not satisfy) and one of only 0, 1 and r - 1."""
    rng = random.Random(100 + log_m)
    for fill in ("full", "half") if log_m > 1 else ("full",):
        cs = domain_circuit(rng.randrange(1 << 30), log_m, fill)
        pk, _, pkb = key_and_oracle(ctx, cs, [rng.randrange(1, R) for _ in range(5)])
        wits = [cs.random_witness(rng)] + ([cs.random_witness(rng, edges_only=True)] if log_m <= 18 else [])
        ref = cport.Prover(cs, pkb)
        PK = ob.ProvingKey(ctx, pk)
        try:
            for i, w in enumerate(wits):
                wb = cport.frs(w)
                assert PK.h_evals(wb) == ref.h_evals(wb), (fill, i)
        finally:
            PK.close()


# ---- C. proofs at real sizes ----------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("log_m", [12, 16, 18])
def test_generic_proofs_at_scale_match_oracle(ctx, log_m):
    """Two proofs of a satisfiable circuit with 2^log_m / 4 outputs, byte for byte against cport.Prover.prove_batch; both
    verify, and fail with a public input changed.  At 2^16 the library's key is also compared with cport.setup_bytes."""
    rng = random.Random(200 + log_m)
    m = 1 << log_m
    cs = CsrCircuit(log_m, 3, 256, m // 4, m - 3 - 1 - rng.randrange(m // 8))
    assert g16.domain_log(cs.n_constraints, cs.n_pub) == log_m
    tw = [rng.randrange(1, R) for _ in range(5)]
    pk, vk, pkb = key_and_oracle(ctx, cs, tw)
    if log_m == 16:
        opkb, ovkb = cport.setup_bytes(cs.as_r1cs(), *tw)
        assert pk == pk_blob(cs, opkb, 0) and vk == vk_blob(ovkb, cs.n_pub)
    wits = [cs.witness(rng) for _ in range(2)]
    wb, rs = b"".join(cport.frs(w) for w in wits), rand_rs(rng, 2)
    PK = ob.ProvingKey(ctx, pk)
    try:
        proofs = PK.prove_witnesses(wb, rs)
    finally:
        PK.close()
    assert proofs == cport.Prover(cs, pkb).prove_batch(wb, rs)
    check_proofs(vk, cs, wits, proofs)


@pytest.mark.gpu
def test_generic_proofs_at_2_20_in_budget_chunks_on_two_lanes(monkeypatch):
    """At 2^20 the lane budget sets the default chunk below 1024.  chunk + 1 proofs run as two chunks on two lanes; every
    proof verifies, and the first and last are the bytes proved one at a time on one lane."""
    import torch
    monkeypatch.delenv("OG_CHUNK", raising=False)
    monkeypatch.delenv("OG_LANES", raising=False)
    rng = random.Random(220)
    m = 1 << 20
    cs = CsrCircuit(20, 3, 512, 1 << 14, m - 3 - 1 - 1000)
    with own_context() as c:          # two budget-sized lanes: scratch of its own, released at the end
        pk, vk, _ = key_and_oracle(c, cs, [rng.randrange(1, R) for _ in range(5)])
        PK = ob.ProvingKey(c, pk)
        try:
            one, plan = PK.prover_plan(1), PK.prover_plan(1 << 20)
            chunk = plan["chunk"]
            assert chunk == LANE_BUDGET // one["scratch_bytes_per_lane"] and 1 <= chunk < 1024 and plan["lanes"] == 2
            batch = chunk + 1
            plan = PK.prover_plan(batch)
            assert (plan["chunk"], plan["lanes"]) == (chunk, 2) and plan["scratch_bytes_per_lane"] <= LANE_BUDGET
            need = 2 * plan["scratch_bytes_per_lane"] * 9 // 8 + 32 * batch * (cs.n_vars + 2) * 9 // 8 + 2 * GIB
            free = torch.cuda.mem_get_info()[0]
            if free < need:
                pytest.skip(f"needs ~{need / GIB:.1f} GiB of free device memory for two lanes at 2^20, {free / GIB:.1f} GiB free")
            distinct = [cs.witness(rng) for _ in range(4)]
            wits = [distinct[0]] + [distinct[1 + i % 2] for i in range(batch - 2)] + [distinct[3]]
            wb, rs = b"".join(cport.frs(w) for w in wits), rand_rs(rng, batch)
            proofs = PK.prove_witnesses(wb, rs)
            check_proofs(vk, cs, wits, proofs)
            monkeypatch.setenv("OG_CHUNK", "1")
            monkeypatch.setenv("OG_LANES", "1")
            ends = PK.prove_witnesses(cport.frs(wits[0]) + cport.frs(wits[-1]), rs[:64] + rs[-64:])
            assert ends == proofs[:256] + proofs[-256:]
        finally:
            PK.close()


# ---- D. degenerate key shapes ---------------------------------------------------------------------------------------------
SHAPES = {
    # name: CsrCircuit arguments (n_pub, n_in, n_out, n_constraints, ...)
    "all-public": (dict(n_pub=24, n_in=16, n_out=8, n_constraints=40), "no private variable: the L query is empty"),
    "all-public-empty-b": (dict(n_pub=12, n_in=12, n_out=0, n_constraints=20, empty_b=True), "n_priv = n_supp = 0"),
    "empty-b": (dict(n_pub=2, n_in=12, n_out=0, n_constraints=30, empty_b=True), "n_supp = 0: the B MSM is beta2, delta2"),
    "max-public": (dict(n_pub=1 << 16, n_in=1 << 16, n_out=64, n_constraints=2000), "n_pub = 2^16, log_m = 17"),
    "heavy-row": (dict(n_pub=3, n_in=6000, n_out=40, n_constraints=300, heavy=5000), "5000 terms in one row of A and B"),
    "duplicate-variable": (dict(n_pub=2, n_in=10, n_out=20, n_constraints=60, duplicate=True), "one variable twice in a row"),
    "one-in-every-row": (dict(n_pub=2, n_in=10, n_out=30, n_constraints=500, one_in_every_row=True), "a heavy column"),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(SHAPES))
def test_degenerate_key_shapes(ctx, name):
    """Keys of unusual shape: proofs byte for byte against the oracle, verified, and refused with a public input changed."""
    kw, _ = SHAPES[name]
    rng = random.Random(name)
    cs = CsrCircuit(name, **kw)
    n_priv = cs.n_vars - cs.n_pub - 1
    assert (n_priv == 0) == name.startswith("all-public")
    pk, vk, pkb = key_and_oracle(ctx, cs, [rng.randrange(1, R) for _ in range(5)])
    if kw.get("empty_b"):
        assert pkb["b1"] == bytes(64 * cs.n_vars) and pkb["b2"] == bytes(128 * cs.n_vars)     # no B support
    else:
        assert pkb["b1"] != bytes(64 * cs.n_vars)
    if name == "max-public":
        assert g16.domain_log(cs.n_constraints, cs.n_pub) == 17
    batch = 1 if name == "max-public" else 3
    wits = [cs.witness(rng, pub_below=1 << 16 if name == "max-public" else R) for _ in range(batch)]
    wb, rs = b"".join(cport.frs(w) for w in wits), rand_rs(rng, batch)
    PK = ob.ProvingKey(ctx, pk)
    try:
        proofs = PK.prove_witnesses(wb, rs)
    finally:
        PK.close()
    assert proofs == cport.Prover(cs, pkb).prove_batch(wb, rs)
    check_proofs(vk, cs, wits, proofs)


# ---- E. the chunk is bounded by the grid --------------------------------------------------------------------------------
@pytest.mark.gpu
def test_chunk_is_bounded_by_the_grid(ctx, monkeypatch):
    """OG_CHUNK above 65535 / 3 on a tiny key: the prover's NTT puts 3 transforms per proof on grid.y, so the chunk is
    clamped to 21845.  30 000 proofs at OG_CHUNK=30000 are the bytes of the default chunking, and every thousandth is the
    oracle's."""
    monkeypatch.delenv("OG_LANES", raising=False)
    rng = random.Random(300)
    cs = CsrCircuit(300, 1, 3, 8, 10)
    pk, vk, pkb = key_and_oracle(ctx, cs, [rng.randrange(1, R) for _ in range(5)])
    batch = 30000
    distinct = [cs.witness(rng) for _ in range(7)]
    wits = [distinct[i % 7] for i in range(batch)]
    wb = b"".join(cport.frs(w) for w in wits)
    rs = rand_rs(rng, batch)
    PK = ob.ProvingKey(ctx, pk)
    try:
        monkeypatch.setenv("OG_CHUNK", "30000")
        big = PK.prove_witnesses(wb, rs)
        assert PK.prover_plan(batch)["chunk"] == GRID_Y_MAX // 3
        monkeypatch.delenv("OG_CHUNK")
        assert PK.prover_plan(batch)["chunk"] == 1024
        assert PK.prove_witnesses(wb, rs) == big
    finally:
        PK.close()
    ref = cport.Prover(cs, pkb)
    picks = range(0, batch, 1000)
    assert b"".join(big[256 * i:256 * i + 256] for i in picks) == ref.prove_batch(
        b"".join(cport.frs(wits[i]) for i in picks), b"".join(rs[64 * i:64 * i + 64] for i in picks))
    check_proofs(vk, cs, [wits[0], wits[-1]], big[:256] + big[-256:])
