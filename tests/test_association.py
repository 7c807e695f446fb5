"""The association-set withdraw statement (oracle/association_circuit.py == csrc/withdraw_circuit.hpp: AssociationBuilder): its
spec, the library's R1CS export, GPU witness, setup, ceremony key and batched prover against the oracle, and a deposit ->
pool tree + association tree -> withdrawal chain."""
import hashlib
import json
import os
import random
import struct

import pytest

import owshen_b200 as ob
from owshen_b200 import api
from oracle import association_circuit as ac
from oracle import bn254 as bn
from oracle import cport, mimc7
from oracle import groth16 as g16
from oracle import withdraw_circuit as wc
from tests.helpers import pk_blob, vk_blob

R = bn.R
GOLD = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "association_vectors.json")))
GIB = 1 << 30
LANE_BUDGET = 28 * GIB          # csrc/groth16.cu: LANE_SCRATCH_BUDGET


# ---- rows: one proof's inputs as ints ---------------------------------------------------------------------------------------
def row(nullifier, secret, recipient, sibs, bits, asibs, abits):
    """bits / abits: path words, bit l set when the level-l node is a right child."""
    return dict(nullifier=nullifier, secret=secret, recipient=recipient, sibs=sibs, bits=bits, asibs=asibs, abits=abits)


def bit_list(word, depth):
    return [(word >> l) & 1 for l in range(depth)]


def bit_word(bits):
    return sum(b << l for l, b in enumerate(bits))


def spec_witness(r):
    d = len(r["sibs"])
    return ac.witness(r["nullifier"], r["secret"], r["recipient"], r["sibs"], bit_list(r["bits"], d), r["asibs"],
                      bit_list(r["abits"], d))


def path(tree, i):
    sibs, bits = tree.path(i)
    return sibs, bit_word(bits)


def valid_rows(rng, batch, depth):
    """Rows whose note is a leaf of its pool tree and of an association tree over a subset, at different indices."""
    rows = []
    for _ in range(batch):
        n, s = rng.randrange(R), rng.randrange(R)
        cm = mimc7.multi_hash([n, s])
        pool, assoc = mimc7.MerkleTree(depth), mimc7.MerkleTree(depth)
        for _ in range(rng.randrange(1, 3)):
            pool.insert(rng.randrange(R))
        i = pool.insert(cm)
        j = assoc.insert(cm)
        assoc.insert(rng.randrange(R))
        rows.append(row(n, s, rng.randrange(1 << 160), *path(pool, i), *path(assoc, j)))
    return rows


def random_rows(rng, batch, depth):
    """Rows of uniformly random inputs (their witnesses satisfy the R1CS too: both roots are derived)."""
    return [row(rng.randrange(R), rng.randrange(R), rng.randrange(R), [rng.randrange(R) for _ in range(depth)], rng.randrange(1 << depth),
                [rng.randrange(R) for _ in range(depth)], rng.randrange(1 << depth)) for _ in range(batch)]


def pack(rows):
    """The seven input buffers of og_association_witness / og_groth16_prove_association."""
    f = cport.frs
    return (f([r["nullifier"] for r in rows]), f([r["secret"] for r in rows]), f([r["recipient"] for r in rows]),
            f([x for r in rows for x in r["sibs"]]), [r["bits"] for r in rows],
            f([x for r in rows for x in r["asibs"]]), [r["abits"] for r in rows])


def oracle_witnesses(rows):
    return b"".join(cport.frs(spec_witness(r)) for r in rows)


def set_env(monkeypatch, **env):
    for k in ("OG_CHUNK", "OG_LANES", "OG_C_A", "OG_C_B", "OG_C_C", "OG_WINDOW_BITS"):
        if env.get(k) is None:
            monkeypatch.delenv(k, raising=False)
        else:
            monkeypatch.setenv(k, str(env[k]))


def failing(cs, w):
    ev = wc.lc_eval
    return [k for k, (a, b, c) in enumerate(zip(cs.A, cs.B, cs.C)) if ev(a, w) * ev(b, w) % R != ev(c, w)]


# ---- CPU: the spec -------------------------------------------------------------------------------------------------------
def test_association_sizes():
    for depth in (1, 2, 32):
        L = ac.Layout(depth)
        assert (L.n_vars, L.n_constraints) == (1101 + 1464 * depth, 1097 + 1462 * depth)
    expect = {32: (47949, 47881, 16), 2: (4029, 4021, 12), 1: (2565, 2559, 12)}
    for depth, (nv, nc, log_m) in expect.items():
        cs = ac.build_r1cs(depth)
        assert (cs.n_vars, cs.n_constraints, cs.n_pub) == (nv, nc, 4), depth
        assert g16.domain_log(cs.n_constraints, cs.n_pub) == log_m, depth
        assert ob.association_r1cs_info(depth) == dict(n_constraints=nc, n_vars=nv, n_pub=4, log_m=log_m), depth
    for bad in (0, 33):
        with pytest.raises(ob.OwshenB200Error):
            ob.association_r1cs_info(bad)


@pytest.fixture(scope="module")
def cs2():
    return ac.build_r1cs(2)


def test_association_witnesses_satisfy(cs2):
    rng = random.Random(1)
    n, s = rng.randrange(R), rng.randrange(R)
    cm = mimc7.multi_hash([n, s])
    pool = mimc7.MerkleTree(2)
    for _ in range(3):
        pool.insert(rng.randrange(R))
    i = pool.insert(cm)                                    # index 3 in the pool
    subset = mimc7.MerkleTree(2)
    subset.insert(rng.randrange(R))
    j = subset.insert(cm)                                  # index 1 in the subset
    only = mimc7.MerkleTree(2)
    k = only.insert(cm)                                    # a subset that holds only this note
    cases = {"different indices": (pool, i, subset, j), "only the note": (pool, i, only, k), "identical trees": (pool, i, pool, i)}
    for name, (t0, i0, t1, i1) in cases.items():
        r = row(n, s, rng.randrange(1 << 160), *path(t0, i0), *path(t1, i1))
        w = spec_witness(r)
        assert cs2.is_satisfied(w), name
        assert (w[ac.V_ROOT], w[ac.V_AROOT]) == (t0.root(), t1.root()), name
    for x in (0, R - 1):
        cm = mimc7.multi_hash([x, x])
        t0, t1 = mimc7.MerkleTree(2), mimc7.MerkleTree(2)
        t0.insert(x); i0 = t0.insert(cm)
        i1 = t1.insert(cm)
        w = spec_witness(row(x, x, x, *path(t0, i0), *path(t1, i1)))
        assert cs2.is_satisfied(w) and w[ac.V_RSQ] == x * x % R, x


def test_association_public_prefix_is_withdraws():
    rng = random.Random(2)
    for depth in (1, 2):
        for r in valid_rows(rng, 2, depth) + random_rows(rng, 2, depth):
            w = spec_witness(r)
            ww = wc.witness(r["nullifier"], r["secret"], r["recipient"], r["sibs"], bit_list(r["bits"], depth))
            assert w[1:4] == ww[1:4]
            assert w[ac.V_NHASH] == mimc7.multi_hash([r["nullifier"]], key=1)
            assert w[ac.Layout(depth).cm_out] == mimc7.multi_hash([r["nullifier"], r["secret"]])


def test_association_mutations_are_unsatisfied(cs2):
    rng = random.Random(3)
    L = ac.Layout(2)
    base = valid_rows(rng, 1, 2)[0]
    w0 = spec_witness(base)
    assert cs2.is_satisfied(w0)

    def mutated(**kw):
        w = list(w0)
        for var, val in kw.items():
            w[int(var[1:])] = val
        return w

    lv = L.level(ac.ASSOC, 1)
    # an association sibling or bit changed (the rest of the assignment kept)
    assert not cs2.is_satisfied(mutated(**{f"v{lv['sib']}": (w0[lv["sib"]] + 1) % R}))
    assert not cs2.is_satisfied(mutated(**{f"v{lv['bit']}": 1 - w0[lv["bit"]]}))
    # a non-boolean bit: its boolean row fails
    w = list(w0)
    lv0 = L.level(ac.ASSOC, 0)
    w[lv0["bit"]] = 2
    bad = failing(cs2, w)
    assert any(cs2.A[k] == {lv0["bit"]: 1} and not cs2.C[k] for k in bad)
    # the public roots
    assert failing(cs2, mutated(**{f"v{ac.V_AROOT}": (w0[ac.V_AROOT] + 1) % R})) == [cs2.n_constraints - 1]
    bad = failing(cs2, mutated(**{f"v{ac.V_ROOT}": (w0[ac.V_ROOT] + 1) % R}))
    assert len(bad) == 1 and cs2.A[bad[0]].get(ac.V_ROOT) == R - 1
    # recipient_sq and nullifier_hash
    assert failing(cs2, mutated(**{f"v{ac.V_RSQ}": (w0[ac.V_RSQ] + 1) % R})) == [0]
    bad = failing(cs2, mutated(**{f"v{ac.V_NHASH}": (w0[ac.V_NHASH] + 1) % R}))
    assert len(bad) == 1 and cs2.C[bad[0]] == {ac.V_NHASH: 1}
    # a note absent from the subset: the path of another leaf yields a root that is not the published one; a witness that
    # claims the published root anyway does not satisfy the R1CS
    n, s = rng.randrange(R), rng.randrange(R)
    cm = mimc7.multi_hash([n, s])
    pool, subset = mimc7.MerkleTree(2), mimc7.MerkleTree(2)
    i = pool.insert(cm)
    subset.insert(rng.randrange(R)); subset.insert(rng.randrange(R))
    r = row(n, s, 5, *path(pool, i), *path(subset, 1))
    w = spec_witness(r)
    assert cs2.is_satisfied(w) and w[ac.V_AROOT] != subset.root()
    w[ac.V_AROOT] = subset.root()
    assert failing(cs2, w) == [cs2.n_constraints - 1]


def test_association_r1cs_export_matches_spec():
    for depth in (1, 2, 32):
        cs = ac.build_r1cs(depth)
        for m in "ABC":
            assert ob.association_r1cs_export(depth, m) == cs.csr(m), (depth, m)


def golden_row(g):
    return row(int(g["nullifier"]), int(g["secret"]), int(g["recipient"]), [int(x) for x in g["siblings"]], g["path_bits"],
               [int(x) for x in g["assoc_siblings"]], g["assoc_path_bits"])


def test_association_golden_proof_reproduced_by_c_port():
    g = GOLD
    cs = ac.build_r1cs(g["depth"])
    pkb, vkb = cport.setup_bytes(cs, *[int(x) for x in g["toxic"]])
    assert hashlib.sha256(pkb["a"] + pkb["b1"] + pkb["b2"] + pkb["l"] + pkb["h"]).hexdigest() == g["pk_queries_sha256"]
    v = g["vk"]
    assert (vkb["alpha1"] + vkb["beta2"] + vkb["gamma2"] + vkb["delta2"] + vkb["ic"]).hex() == v["alpha1"] + v["beta2"] + v["gamma2"] + v["delta2"] + v["ic"]
    w = spec_witness(golden_row(g))
    assert cs.is_satisfied(w)
    wit = cport.frs(w)
    assert hashlib.sha256(wit).hexdigest() == g["witness_sha256"]
    assert cport.unfr(wit[32:32 * 5]) == [int(x) for x in g["public"]]
    assert cport.Prover(cs, pkb).prove(wit, int(g["r"]), int(g["s"])).hex() == g["proof"]
    assert ob.verify(vk_blob(vkb, 4), wit[32:32 * 5], bytes.fromhex(g["proof"]))


# ---- GPU -----------------------------------------------------------------------------------------------------------------
_KEYS = {}


def association_keys(ctx, depth):
    """(pk, vk, r1cs, oracle pk bytes, oracle vk bytes) of the depth-`depth` association statement, made once per process."""
    if depth not in _KEYS:
        rng = random.Random(60 + depth)
        tw = [rng.randrange(1, R) for _ in range(5)]
        pk, vk = ob.setup_association(ctx, depth, *tw)
        cs = ac.build_r1cs(depth)
        pkb, vkb = cport.setup_bytes(cs, *tw)
        _KEYS[depth] = (pk, vk, cs, pkb, vkb)
    return _KEYS[depth]


def proofs_verify(vk, proofs, pub, batch):
    return [ob.verify(vk, pub[128 * i:128 * i + 128], proofs[256 * i:256 * i + 256]) for i in range(batch)]


@pytest.mark.gpu
def test_association_witness_matches_oracle(ctx):
    rng = random.Random(61)
    for depth, n_random in ((2, 37), (32, 4)):
        rows = random_rows(rng, n_random, depth) + valid_rows(rng, 3, depth)
        assert ctx.association_witness(depth, *pack(rows)) == oracle_witnesses(rows), depth
    # edge values: field inputs 0 and r - 1 everywhere, path words 0 and all ones, at depth 2 and 32
    for depth in (2, 32):
        rows = [row(x, x, x, [x] * depth, b, [x] * depth, (1 << depth) - 1 - b) for x in (0, R - 1) for b in (0, (1 << depth) - 1)]
        assert ctx.association_witness(depth, *pack(rows)) == oracle_witnesses(rows), depth
    rows = valid_rows(rng, 2, 2)
    # a field input >= r in any of the five field arrays
    for k in (0, 1, 2, 3, 5):
        p = list(pack(rows))
        p[k] = R.to_bytes(32, "little") + p[k][32:]
        with pytest.raises(ob.OwshenB200Error) as e:
            ctx.association_witness(2, *p)
        assert e.value.code == -4 or "encoding" in str(e.value).lower(), k
    # wrong lengths
    p = pack(rows)
    for k, bad in ((3, p[3][:-32]), (4, p[4][:1]), (5, p[5] + bytes(32)), (6, p[6] + [0]), (2, p[2][:32])):
        q = list(p)
        q[k] = bad
        with pytest.raises(ValueError):
            ctx.association_witness(2, *q)


@pytest.mark.gpu
def test_setup_association_matches_oracle(ctx):
    for depth in (2, 32):
        pk, vk, cs, pkb, vkb = association_keys(ctx, depth)
        assert pk == pk_blob(cs, pkb, 0), depth
        assert vk == vk_blob(vkb, 4), depth


@pytest.mark.gpu
def test_association_key_from_ceremony(ctx):
    """One phase-1 contribution (t, a, b), then the depth-2 key: before phase 2, gamma = delta = 1 (DESIGN.md section 4b)."""
    rng = random.Random(62)
    t, a, b = (rng.randrange(1, R) for _ in range(3))
    acc0 = ob.ptau_new(ctx, 12)                           # the depth-2 association domain is 2^12
    acc1, rec = ob.ptau_contribute(ctx, acc0, [t, a, b], [rng.randrange(1, R) for _ in range(3)])
    assert ob.ptau_verify(ctx, acc0, acc1, rec)
    pk, vk = ob.ptau_prepare_association(ctx, acc1, 2)
    assert (pk, vk) == ob.setup_association(ctx, 2, t, a, b, 1, 1)
    PK = ob.ProvingKey(ctx, pk)
    try:
        assert PK.association_depth == 2
    finally:
        PK.close()


@pytest.mark.gpu
@pytest.mark.parametrize("depth,batch", [(2, 40), (32, 3)])
def test_prove_association_matches_oracle(ctx, monkeypatch, depth, batch):
    pk, vk, cs, pkb, vkb = association_keys(ctx, depth)
    rng = random.Random(63 + depth)
    rows = valid_rows(rng, batch, depth)
    rs = cport.frs([rng.randrange(R) for _ in range(2 * batch)])
    wit = oracle_witnesses(rows)
    exp = cport.Prover(cs, pkb).prove_batch(wit, rs)
    results = []
    for env in (dict(), dict(OG_CHUNK=3, OG_LANES=1), dict(OG_CHUNK=3, OG_LANES=2)):
        set_env(monkeypatch, **env)
        PK = ob.ProvingKey(ctx, pk)
        try:
            assert (PK.n_vars, PK.n_pub, PK.depth, PK.association_depth, PK.transfer_depth) == (cs.n_vars, 4, 0, depth, None)
            results.append(PK.prove_association(*pack(rows), rs))
        finally:
            PK.close()
    set_env(monkeypatch)
    nv = cs.n_vars
    for proofs, pub in results:
        assert proofs == exp
        assert pub == b"".join(wit[32 * nv * i + 32:32 * nv * i + 32 * 5] for i in range(batch))
    proofs, pub = results[0]
    assert all(proofs_verify(vk, proofs, pub, batch))
    bad = bytearray(pub[:128]); bad[96] ^= 1          # another association root
    assert not ob.verify(vk, bytes(bad), proofs[:256])


@pytest.mark.gpu
def test_prove_association_dev_matches_host_entry_point(ctx):
    import torch
    pk = association_keys(ctx, 2)[0]
    rng = random.Random(64)
    batch = 5
    rows = valid_rows(rng, batch, 2)
    rs = cport.frs([rng.randrange(R) for _ in range(2 * batch)])
    p = pack(rows)
    PK = ob.ProvingKey(ctx, pk)
    try:
        proofs, pub = PK.prove_association(*p, rs)
        words = lambda xs: struct.pack(f"<{len(xs)}I", *xs)
        dev = lambda b: torch.frombuffer(bytearray(b), dtype=torch.uint8).to("cuda")
        d_in = [dev(x) for x in (p[0], p[1], p[2], p[3], words(p[4]), p[5], words(p[6]), rs)]
        d_pr = torch.zeros(256 * batch, dtype=torch.uint8, device="cuda")
        d_pub = torch.zeros(128 * batch, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        rc = api.lib().og_groth16_prove_association_dev(ctx._h, PK._h, *[api._ptr(t) for t in d_in[:7]], batch, api._ptr(d_in[7]),
                                                        api._ptr(d_pr), api._ptr(d_pub))
        assert rc == 0
        ctx.sync()
        assert bytes(d_pr.cpu().numpy()) == proofs and bytes(d_pub.cpu().numpy()) == pub
    finally:
        PK.close()


@pytest.mark.gpu
def test_association_golden_proof(ctx):
    g = GOLD
    pk, vk = ob.setup_association(ctx, g["depth"], *[int(x) for x in g["toxic"]])
    v = g["vk"]
    assert vk[12:].hex() == v["alpha1"] + v["beta2"] + v["gamma2"] + v["delta2"] + v["ic"]
    rs = bn.fr_to_bytes(int(g["r"])) + bn.fr_to_bytes(int(g["s"]))
    PK = ob.ProvingKey(ctx, pk)
    try:
        proofs, pub = PK.prove_association(*pack([golden_row(g)]), rs)
    finally:
        PK.close()
    assert proofs.hex() == g["proof"]
    assert cport.unfr(pub) == [int(x) for x in g["public"]]
    assert ob.verify(vk, pub, proofs)


@pytest.mark.gpu
def test_note_missing_from_subset_fails_alone(ctx):
    """A row whose association path comes from another leaf is proved like any other; checked against the published roots,
    its proof fails and the rest of the batch verifies."""
    pk, vk = association_keys(ctx, 2)[:2]
    rng = random.Random(65)
    rows = valid_rows(rng, 8, 2)
    published = [(r, spec_witness(r)) for r in rows]
    roots = [(w[ac.V_ROOT], w[ac.V_AROOT]) for _, w in published]
    # row 3: its note is not in the subset tree; the path is that of the subset's other leaf
    r = rows[3]
    subset = mimc7.MerkleTree(2)
    subset.insert(rng.randrange(R)); subset.insert(rng.randrange(R))
    r["asibs"], r["abits"] = path(subset, 1)
    roots[3] = (roots[3][0], subset.root())
    rs = cport.frs([rng.randrange(R) for _ in range(16)])
    PK = ob.ProvingKey(ctx, pk)
    try:
        proofs, pub = PK.prove_association(*pack(rows), rs)
    finally:
        PK.close()
    assert cport.unfr(pub[128 * 3 + 96:128 * 4]) != [subset.root()]
    ok = []
    for i, (root, aroot) in enumerate(roots):
        p = cport.unfr(pub[128 * i:128 * i + 128])
        ok.append(ob.verify(vk, cport.frs([root, p[1], p[2], aroot]), proofs[256 * i:256 * i + 256]))
    assert ok == [i != 3 for i in range(8)]


def _generic_key(ctx, n_vars, n_pub, rng):
    cs = wc.R1CS(n_vars, n_pub)
    for j in range(n_vars - 1):
        cs.add({j: 1}, {j: 1}, {j + 1: 1})
    return ob.setup_r1cs(ctx, cs.n_vars, cs.n_pub, cs.csr("A"), cs.csr("B"), cs.csr("C"), *[rng.randrange(1, R) for _ in range(5)])[0]


@pytest.mark.gpu
def test_association_and_other_provers_refuse_each_others_keys(ctx):
    import torch
    d_buf = torch.zeros(1 << 16, dtype=torch.uint8, device="cuda")
    d = api._ptr(d_buf)      # every device argument of the _dev entry points
    rng = random.Random(66)
    pk_a = association_keys(ctx, 2)[0]
    rows = random_rows(rng, 2, 2)
    p = pack(rows)
    rs = cport.frs([rng.randrange(R) for _ in range(4)])
    tw = [rng.randrange(1, R) for _ in range(5)]
    nv2 = ac.Layout(2).n_vars
    others = [ob.setup_withdraw(ctx, 2, *tw)[0], ob.setup_deposit(ctx, *tw)[0], ob.setup_transfer(ctx, 2, *tw)[0],
              _generic_key(ctx, nv2, 4, rng), _generic_key(ctx, nv2, 3, rng)]
    bits, abits = (api.C.c_uint32 * 2)(*p[4]), (api.C.c_uint32 * 2)(*p[6])
    args = [p[0], p[1], p[2], p[3], bits, p[5], abits]
    for pk in others:
        PK = ob.ProvingKey(ctx, pk)
        try:
            with pytest.raises(ob.OwshenB200Error) as e:
                PK.prove_association(*p, rs)
            assert e.value.code == api.OG_E_INVALID
            for b in (2, 0):      # the key is wrong whatever the batch
                rc = api.lib().og_groth16_prove_association(ctx._h, PK._h, *[api._ptr(x) for x in args], b, rs,
                                                            api.C.create_string_buffer(512), None)
                assert rc == api.OG_E_INVALID, b
                assert api.lib().og_groth16_prove_association_dev(ctx._h, PK._h, *[d] * 7, b, d, d, None) == api.OG_E_INVALID, b
        finally:
            PK.close()
    PK = ob.ProvingKey(ctx, pk_a)
    try:
        nul, sec, rec = p[0], p[1], p[2]
        for b in (2, 0):
            rc = api.lib().og_groth16_prove_withdraw(ctx._h, PK._h, nul, sec, rec, bytes(128), (api.C.c_uint32 * 2)(0, 0), b, rs,
                                                     api.C.create_string_buffer(512), None)
            assert rc == api.OG_E_INVALID, b
            assert api.lib().og_groth16_prove_withdraw_dev(ctx._h, PK._h, d, d, d, d, d, b, d, d, None) == api.OG_E_INVALID, b
        with pytest.raises(ob.OwshenB200Error) as e:
            PK.prove_deposit(nul, sec, rec, rs)
        assert e.value.code == api.OG_E_INVALID
        with pytest.raises(ob.OwshenB200Error) as e:
            PK.prove_transfer(cport.frs([1, 2]), cport.frs([3, 4]), rec, bytes(128), bytes(128), [0] * 4, bytes(256), [0] * 4,
                              bytes(128), bytes(128), [0] * 4, rs)
        assert e.value.code == api.OG_E_INVALID
        t_args = [bytes(64), bytes(64), bytes(64), bytes(128), bytes(128), bytes(32), bytes(256), (api.C.c_uint32 * 4)(),
                  bytes(128), bytes(128), bytes(32)]
        rc = api.lib().og_groth16_prove_transfer(ctx._h, PK._h, *[api._ptr(x) for x in t_args], 2, rs, api.C.create_string_buffer(512), None)
        assert rc == api.OG_E_INVALID
        assert len(PK.prove_association(*p, rs)[0]) == 512          # the context is still usable
    finally:
        PK.close()


@pytest.mark.gpu
def test_deposit_to_association_withdraw_chain(ctx):
    """Deposits proved with prove_deposit, their commitments in a depth-32 pool tree and a strict subset of them in an
    association set provider's tree (both GPU MerkleTrees); depth-32 association withdrawals of the subset's notes verify
    against both published roots, and the note left out of the subset cannot produce one."""
    rng = random.Random(67)
    tw = [rng.randrange(1, R) for _ in range(5)]
    pk_d, vk_d = ob.setup_deposit(ctx, *tw)
    n = 5
    notes = [(rng.randrange(R), rng.randrange(R)) for _ in range(n)]
    PK = ob.ProvingKey(ctx, pk_d)
    try:
        proofs, pub = PK.prove_deposit(cport.frs([x[0] for x in notes]), cport.frs([x[1] for x in notes]),
                                       cport.frs([rng.randrange(1 << 160) for _ in range(n)]), cport.frs([rng.randrange(R) for _ in range(2 * n)]))
    finally:
        PK.close()
    assert all(ob.verify(vk_d, pub[64 * i:64 * i + 64], proofs[256 * i:256 * i + 256]) for i in range(n))
    cms = [cport.unfr(pub[64 * i:64 * i + 32])[0] for i in range(n)]
    assert cms == [mimc7.multi_hash(list(x)) for x in notes]
    pool = ob.MerkleTree(ctx, 32)
    pool.insert_batch([rng.randrange(R) for _ in range(3)])
    pool_idx = pool.insert_batch(cms)
    subset = [0, 2, 4]                                     # deposit 1 and 3 are left out
    assoc = ob.MerkleTree(ctx, 32, prefix=b"as/")
    assoc.insert_batch([rng.randrange(R)])
    assoc_idx = dict(zip(subset, assoc.insert_batch([cms[k] for k in subset])))
    as_int = lambda b: int.from_bytes(b, "little")
    roots = (as_int(pool.root()), as_int(assoc.root()))
    pk, vk = association_keys(ctx, 32)[:2]
    rows, recipients = [], [rng.randrange(1 << 160) for _ in range(n)]
    for k in subset + [1]:
        sibs, bits = pool.paths([pool_idx[k]])
        a = assoc_idx.get(k, 1)                             # the left-out note borrows a member's path
        asibs, abits = assoc.paths([a])
        rows.append(row(notes[k][0], notes[k][1], recipients[k], cport.unfr(sibs), bits[0], cport.unfr(asibs), abits[0]))
    PK = ob.ProvingKey(ctx, pk)
    try:
        proofs, pub = PK.prove_association(*pack(rows), cport.frs([rng.randrange(R) for _ in range(2 * len(rows))]))
    finally:
        PK.close()
    for i, k in enumerate(subset + [1]):
        p = cport.unfr(pub[128 * i:128 * i + 128])
        published = cport.frs([roots[0], p[1], p[2], roots[1]])
        nh = wc.witness(notes[k][0], notes[k][1], recipients[k], rows[i]["sibs"], bit_list(rows[i]["bits"], 32))[wc.V_NHASH]
        assert p[1] == nh and p[2] == recipients[k] and p[0] == roots[0], k
        if k in assoc_idx:
            assert p[3] == roots[1] and ob.verify(vk, published, proofs[256 * i:256 * i + 256]), k
        else:
            assert p[3] != roots[1] and not ob.verify(vk, published, proofs[256 * i:256 * i + 256]), k


@pytest.mark.gpu
def test_association_prover_plan_and_batch_above_default_chunk(monkeypatch):
    """The depth-32 key's default chunk is what the 28 GiB lane budget gives; chunk + 1 proofs at default settings run as two
    chunks on two lanes, match the oracle and verify."""
    import torch
    set_env(monkeypatch)
    c = ob.Context(0)          # its own scratch: the session context keeps what earlier tests grew
    try:
        pk, vk, cs, pkb, vkb = association_keys(c, 32)
        PK = ob.ProvingKey(c, pk)
        try:
            one = PK.prover_plan(1)
            plan = PK.prover_plan(1 << 20)
            assert plan["chunk"] == min(1024, LANE_BUDGET // one["scratch_bytes_per_lane"]) and plan["lanes"] == 2
            assert plan["scratch_bytes_per_lane"] <= LANE_BUDGET
            chunk = plan["chunk"]
            batch = chunk + 1
            plan = PK.prover_plan(batch)
            assert plan["lanes"] == 2
            need = 2 * plan["scratch_bytes_per_lane"] * 9 // 8 + 32 * batch * (cs.n_vars + 2) * 9 // 8 + 4 * GIB
            free = torch.cuda.mem_get_info()[0]
            if free < need:
                pytest.skip(f"needs ~{need / GIB:.1f} GiB of free device memory for {batch} depth-32 proofs on two lanes, "
                            f"{free / GIB:.1f} GiB free")
            rng = random.Random(68)
            rows = valid_rows(rng, 2, 32)
            rows = [rows[0]] + random_rows(rng, batch - 2, 32) + [rows[1]]
            rs = cport.frs([rng.randrange(R) for _ in range(2 * batch)])
            proofs, pub = PK.prove_association(*pack(rows), rs)
        finally:
            PK.close()
    finally:
        c.close()
    prover = cport.Prover(cs, pkb)
    for i in (0, chunk - 1, chunk):
        wit = cport.frs(spec_witness(rows[i]))
        assert proofs[256 * i:256 * i + 256] == prover.prove_batch(wit, rs[64 * i:64 * i + 64]), i
        assert ob.verify(vk, pub[128 * i:128 * i + 128], proofs[256 * i:256 * i + 256]), i
