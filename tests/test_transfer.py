"""The transfer statement (oracle/transfer_circuit.py == csrc/withdraw_circuit.hpp: TransferBuilder): its spec, the library's
R1CS export, GPU witness, setup and batched prover against the oracle, a deposit -> transfer -> withdrawal chain through one
tree, and the prover's default chunk taken from the key's scratch."""
import hashlib
import json
import os
import random
import struct

import pytest

import owshen_b200 as ob
from owshen_b200 import api
from oracle import bn254 as bn
from oracle import cport, mimc7
from oracle import groth16 as g16
from oracle import transfer_circuit as tc
from oracle import withdraw_circuit as wc
from tests.helpers import pk_blob, vk_blob, withdraw_keys32

R = bn.R
U64 = (1 << 64) - 1
GOLD = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "transfer_vectors.json")))
GIB = 1 << 30
LANE_BUDGET = 28 * GIB          # csrc/groth16.cu: LANE_SCRATCH_BUDGET


# ---- rows: one transfer's inputs as ints ------------------------------------------------------------------------------------
def row(root, token, recipient, ins, outs):
    """ins: two (nullifier, secret, amount, siblings, path_bits); outs: two (nullifier, secret, amount)."""
    return dict(root=root, token=token, recipient=recipient, ins=ins, outs=outs)


def spec_witness(r):
    return tc.witness(r["root"], r["token"], r["recipient"], r["ins"], r["outs"])


def valid_rows(rng, batch, depth, amounts=None, token=None):
    """Rows whose input notes are leaves of one tree (a tree per row when the batch's notes do not fit in one), so every
    row satisfies the statement.  amounts: per row (in0, in1, out0, out1), default random."""
    per_row = 2 * batch + 1 > 1 << depth
    tree, rows, pending = None, [], []
    for k in range(batch):
        if tree is None or per_row:
            tree = mimc7.MerkleTree(depth)
            tree.insert(rng.randrange(R))       # another note first
        tok = rng.randrange(R) if token is None else token
        a = amounts[k] if amounts else [rng.randrange(1 << 64) for _ in range(4)]
        notes = [(rng.randrange(R), rng.randrange(R), a[i]) for i in range(2)]
        idx = [tree.insert(mimc7.multi_hash([n, s, tok, am])) for n, s, am in notes]
        outs = [(rng.randrange(R), rng.randrange(R), a[2 + j]) for j in range(2)]
        pending.append((tree, idx, notes, tok, outs))
    for tree, idx, notes, tok, outs in pending:
        ins = []
        for (n, s, am), i in zip(notes, idx):
            sibs, bits = tree.path(i)
            ins.append((n, s, am, sibs, sum(b << l for l, b in enumerate(bits))))
        rows.append(row(tree.root(), tok, rng.randrange(1 << 160), ins, outs))
    return rows


def random_rows(rng, batch, depth):
    """Rows of uniformly random inputs (their witnesses do not satisfy the statement: the prover does not care)."""
    return [row(rng.randrange(R), rng.randrange(R), rng.randrange(R),
                [(rng.randrange(R), rng.randrange(R), rng.randrange(1 << 64), [rng.randrange(R) for _ in range(depth)],
                  rng.randrange(1 << depth)) for _ in range(2)],
                [(rng.randrange(R), rng.randrange(R), rng.randrange(1 << 64)) for _ in range(2)]) for _ in range(batch)]


def pack(rows):
    """The eleven input buffers of og_transfer_witness / og_groth16_prove_transfer."""
    f = cport.frs
    u64 = lambda xs: struct.pack(f"<{len(xs)}Q", *xs)
    return (f([r["root"] for r in rows]), f([r["token"] for r in rows]), f([r["recipient"] for r in rows]),
            f([n[0] for r in rows for n in r["ins"]]), f([n[1] for r in rows for n in r["ins"]]),
            u64([n[2] for r in rows for n in r["ins"]]), f([s for r in rows for n in r["ins"] for s in n[3]]),
            [n[4] for r in rows for n in r["ins"]],
            f([n[0] for r in rows for n in r["outs"]]), f([n[1] for r in rows for n in r["outs"]]),
            u64([n[2] for r in rows for n in r["outs"]]))


def oracle_witnesses(rows):
    return b"".join(cport.frs(spec_witness(r)) for r in rows)


def set_env(monkeypatch, **env):
    for k in ("OG_CHUNK", "OG_LANES", "OG_C_A", "OG_C_B", "OG_C_C", "OG_WINDOW_BITS"):
        if env.get(k) is None:
            monkeypatch.delenv(k, raising=False)
        else:
            monkeypatch.setenv(k, str(env[k]))


def failing(cs, w):
    """Indices of the constraints w does not satisfy."""
    ev = wc.lc_eval
    return [k for k, (a, b, c) in enumerate(zip(cs.A, cs.B, cs.C)) if ev(a, w) * ev(b, w) % R != ev(c, w)]


# ---- CPU: the spec -------------------------------------------------------------------------------------------------------
def test_transfer_sizes():
    for depth in (1, 2, 32):
        L = tc.Layout(depth)
        P = L.perm
        assert (L.n_vars, L.n_constraints) == (283 + 18 * P + depth * (4 * P + 8), 273 + 18 * P + depth * (4 * P + 6))
    cs = tc.build_r1cs(32)
    assert (cs.n_vars, cs.n_constraints, cs.n_pub) == (53683, 53609, 8)
    assert g16.domain_log(cs.n_constraints, cs.n_pub) == 16
    cs = tc.build_r1cs(2)
    assert (cs.n_vars, cs.n_constraints) == (9763, 9749) and g16.domain_log(cs.n_constraints, cs.n_pub) == 14
    for depth in (1, 2, 32):
        L = tc.Layout(depth)
        info = ob.transfer_r1cs_info(depth)
        assert info == dict(n_constraints=L.n_constraints, n_vars=L.n_vars, n_pub=8,
                            log_m=g16.domain_log(L.n_constraints, 8)), depth
    for bad in (0, 33):
        with pytest.raises(ob.OwshenB200Error):
            ob.transfer_r1cs_info(bad)


@pytest.fixture(scope="module")
def cs2():
    return tc.build_r1cs(2)


def test_transfer_witnesses_satisfy(cs2):
    rng = random.Random(1)
    cases = {
        "deposit": [(0, 0, 40, 2)],
        "transfer": [(5, 7, 9, 3)],
        "withdrawal with change": [(100, 23, 80, 0)],
        "zero": [(0, 0, 0, 0)], "one": [(1, 1, 1, 1)], "max": [(U64, U64, U64, U64)],
    }
    for name, amounts in cases.items():
        r = valid_rows(rng, 1, 2, amounts)[0]
        if name == "deposit":    # two dummy inputs: no real path, proved against whatever the current root is
            r["ins"] = [(n, s, 0, [rng.randrange(R), rng.randrange(R)], rng.randrange(4)) for n, s, _, _, _ in r["ins"]]
        w = spec_witness(r)
        assert cs2.is_satisfied(w), name
        a = amounts[0]
        assert w[tc.V_PUB_AMOUNT] == (a[2] + a[3] - a[0] - a[1]) % R, name
    w = spec_witness(valid_rows(rng, 1, 2, [(100, 23, 80, 0)])[0])
    assert w[tc.V_PUB_AMOUNT] == R - 43 and w[tc.V_PUB_AMOUNT] > R - (1 << 65)
    # field inputs 0 and r - 1 everywhere a field element goes
    for x in (0, R - 1):
        tree = mimc7.MerkleTree(2)
        notes = [(x, x, 3), ((x + 1) % R, x, 0)]
        for n, s, a in notes:
            tree.insert(mimc7.multi_hash([n, s, x, a]))
        ins = [(n, s, a, tree.path(i)[0], sum(b << l for l, b in enumerate(tree.path(i)[1]))) for i, (n, s, a) in enumerate(notes)]
        w = spec_witness(row(tree.root(), x, x, ins, [(x, x, 1), (x, x, 2)]))
        assert cs2.is_satisfied(w), x


def test_transfer_identities():
    rng = random.Random(2)
    r = valid_rows(rng, 1, 2)[0]
    w = spec_witness(r)
    L = tc.Layout(2)
    for j, (n, s, a) in enumerate(r["outs"]):
        assert w[tc.V_OUT_CM[j]] == mimc7.multi_hash([n, s, r["token"], a]) == w[L.out(j)["cm_out"]]
    for i, (n, s, a, sibs, bits) in enumerate(r["ins"]):
        assert w[tc.V_NH[i]] == mimc7.multi_hash([n], key=1)
        assert w[tc.V_NH[i]] == wc.witness(n, s, 7, sibs, [(bits >> l) & 1 for l in range(2)])[wc.V_NHASH]
        assert w[L.inp(i)["cm_out"]] == mimc7.multi_hash([n, s, r["token"], a])
    d = (w[5] - w[6]) % R
    assert w[tc.V_NH_INV] * d % R == 1


def test_transfer_mutations_are_unsatisfied(cs2):
    rng = random.Random(3)
    L = tc.Layout(2)
    base = valid_rows(rng, 1, 2, [(6, 9, 2, 13)])[0]
    assert cs2.is_satisfied(spec_witness(base))
    # a nonzero input against a wrong root; a zero-valued one needs no path
    r = dict(base, root=(base["root"] + 1) % R)
    assert not cs2.is_satisfied(spec_witness(r))
    r["ins"] = [(n, s, 0, sb, b) for n, s, _, sb, b in base["ins"]]
    r["outs"] = [(1, 2, 0), (3, 4, 0)]
    assert cs2.is_satisfied(spec_witness(r))
    # an amount bit set to 2: out0 = 2 = 0*1 + 1*2 written as 2*1 + 0*2 packs the same amount; only bit 0's boolean row fails
    w = spec_witness(base)
    v = L.out(0)
    assert (w[v["bits"]], w[v["bits"] + 1]) == (0, 1)
    w[v["bits"]], w[v["bits"] + 1] = 2, 0
    bad = failing(cs2, w)
    assert len(bad) == 1 and cs2.A[bad[0]] == {v["bits"]: 1}
    # an amount of 2^64: no 65th bit exists, so the packing row fails (commitment and public amount made consistent)
    w = spec_witness(base)
    w[tc.V_OUT_CM[0]] = tc._note_witness(w, v, 1, 2, base["token"], 1 << 64, L.perm, 91)
    w[v["null"]], w[v["sec"]] = 1, 2
    w[tc.V_PUB_AMOUNT] = ((1 << 64) + 13 - 6 - 9) % R
    bad = failing(cs2, w)
    assert len(bad) == 1 and cs2.A[bad[0]].get(v["amount"]) == R - 1
    # equal nullifiers, with any nh_diff_inv
    r = valid_rows(rng, 1, 2, [(4, 5, 6, 3)])[0]
    n0 = r["ins"][0][0]
    tree = mimc7.MerkleTree(2)
    notes = [(n0, 11, 4), (n0, 12, 5)]
    for n, s, a in notes:
        tree.insert(mimc7.multi_hash([n, s, r["token"], a]))
    r["ins"] = [(n, s, a, tree.path(i)[0], sum(b << l for l, b in enumerate(tree.path(i)[1]))) for i, (n, s, a) in enumerate(notes)]
    r["root"] = tree.root()
    w = spec_witness(r)
    assert w[tc.V_NH[0]] == w[tc.V_NH[1]] and w[tc.V_NH_INV] == 0
    for inv in (0, 1, rng.randrange(R)):
        w[tc.V_NH_INV] = inv
        assert failing(cs2, w) == [cs2.n_constraints - 1]
    # conservation off by one
    w = spec_witness(base)
    w[tc.V_PUB_AMOUNT] = (w[tc.V_PUB_AMOUNT] + 1) % R
    assert failing(cs2, w) == [cs2.n_constraints - 2]
    # an input note committed under another token: its leaf is in the tree, but the statement hashes the public token
    other = (base["token"] + 1) % R
    tree = mimc7.MerkleTree(2)
    tree.insert(mimc7.multi_hash([base["ins"][0][0], base["ins"][0][1], other, 6]))
    tree.insert(mimc7.multi_hash([base["ins"][1][0], base["ins"][1][1], base["token"], 9]))
    r = dict(base, root=tree.root())
    r["ins"] = [(n, s, a, tree.path(i)[0], sum(b << l for l, b in enumerate(tree.path(i)[1])))
                for i, (n, s, a, _, _) in enumerate(base["ins"])]
    assert not cs2.is_satisfied(spec_witness(r))
    r["token"] = other
    assert not cs2.is_satisfied(spec_witness(r))    # and under the other token, input 1 is the stranger


def test_transfer_r1cs_export_matches_spec():
    for depth in (1, 2, 32):
        cs = tc.build_r1cs(depth)
        for m in "ABC":
            assert ob.transfer_r1cs_export(depth, m) == cs.csr(m), (depth, m)


def test_transfer_golden_proof_reproduced_by_c_port():
    g = GOLD
    depth = g["depth"]
    cs = tc.build_r1cs(depth)
    pkb, vkb = cport.setup_bytes(cs, *[int(x) for x in g["toxic"]])
    assert hashlib.sha256(pkb["a"] + pkb["b1"] + pkb["b2"] + pkb["l"] + pkb["h"]).hexdigest() == g["pk_queries_sha256"]
    v = g["vk"]
    assert (vkb["alpha1"] + vkb["beta2"] + vkb["gamma2"] + vkb["delta2"] + vkb["ic"]).hex() == v["alpha1"] + v["beta2"] + v["gamma2"] + v["delta2"] + v["ic"]
    r = golden_row(g)
    w = spec_witness(r)
    assert cs.is_satisfied(w)
    wit = cport.frs(w)
    assert hashlib.sha256(wit).hexdigest() == g["witness_sha256"]
    assert cport.unfr(wit[32:32 * 9]) == [int(x) for x in g["public"]]
    assert cport.Prover(cs, pkb).prove(wit, int(g["r"]), int(g["s"])).hex() == g["proof"]
    assert ob.verify(vk_blob(vkb, 8), wit[32:32 * 9], bytes.fromhex(g["proof"]))


def golden_row(g):
    ins = [(int(n["nullifier"]), int(n["secret"]), int(n["amount"]), [int(x) for x in n["siblings"]], int(n["path_bits"]))
           for n in g["inputs"]]
    outs = [(int(n["nullifier"]), int(n["secret"]), int(n["amount"])) for n in g["outputs"]]
    return row(int(g["root"]), int(g["token"]), int(g["recipient"]), ins, outs)


# ---- GPU -----------------------------------------------------------------------------------------------------------------
_KEYS = {}


def transfer_keys(ctx, depth):
    """(pk, vk, r1cs, oracle pk bytes, oracle vk bytes) of the depth-`depth` transfer statement, made once per process."""
    if depth not in _KEYS:
        rng = random.Random(40 + depth)
        tw = [rng.randrange(1, R) for _ in range(5)]
        pk, vk = ob.setup_transfer(ctx, depth, *tw)
        cs = tc.build_r1cs(depth)
        pkb, vkb = cport.setup_bytes(cs, *tw)
        _KEYS[depth] = (pk, vk, cs, pkb, vkb)
    return _KEYS[depth]


def proofs_verify(vk, proofs, pub, batch):
    return [ob.verify(vk, pub[256 * i:256 * i + 256], proofs[256 * i:256 * i + 256]) for i in range(batch)]


@pytest.mark.gpu
def test_transfer_witness_matches_oracle(ctx):
    rng = random.Random(41)
    for depth in (2, 32):
        rows = random_rows(rng, 37 if depth == 2 else 5, depth) + valid_rows(rng, 3, depth)
        assert ctx.transfer_witness(depth, *pack(rows)) == oracle_witnesses(rows), depth
    # edge values: amounts 0, 1, 2^64 - 1 on every note; field inputs 0 and r - 1; one nullifier in both inputs (inverse 0)
    rows = []
    for a in (0, 1, U64):
        for x in (0, R - 1):
            rows.append(row(x, x, x, [(x, x, a, [x, x], 3), ((x + 1) % R, x, a, [x, x], 0)], [(x, x, a), (x, x, a)]))
    rows.append(row(5, 6, 7, [(9, 1, 2, [3, 4], 1), (9, 2, 3, [5, 6], 2)], [(1, 1, 1), (2, 2, 4)]))
    got = ctx.transfer_witness(2, *pack(rows))
    assert got == oracle_witnesses(rows)
    nv = tc.Layout(2).n_vars
    assert got[32 * nv * (len(rows) - 1) + 32 * tc.V_NH_INV:][:32] == bytes(32)
    # amounts as ints and as numpy arrays give the same bytes
    import numpy as np
    p = list(pack(rows))
    p[5] = [n[2] for r in rows for n in r["ins"]]
    p[10] = np.array([n[2] for r in rows for n in r["outs"]], dtype=np.uint64)
    assert ctx.transfer_witness(2, *p) == got
    # a field input >= r
    for k in (0, 1, 2, 3, 4, 6, 8, 9):
        p = list(pack(rows[:1]))
        p[k] = R.to_bytes(32, "little") + p[k][32:]
        with pytest.raises(ob.OwshenB200Error) as e:
            ctx.transfer_witness(2, *p)
        assert e.value.code == -4 or "encoding" in str(e.value).lower(), k
    with pytest.raises(ValueError):
        ctx.transfer_witness(2, *pack(rows)[:7], [0], *pack(rows)[8:])


@pytest.mark.gpu
def test_setup_transfer_matches_oracle(ctx):
    for depth in (2, 32):
        pk, vk, cs, pkb, vkb = transfer_keys(ctx, depth)
        assert pk == pk_blob(cs, pkb, 0), depth
        assert vk == vk_blob(vkb, 8), depth


@pytest.mark.gpu
@pytest.mark.parametrize("depth,batch", [(2, 40), (32, 3)])
def test_prove_transfer_matches_oracle(ctx, monkeypatch, depth, batch):
    pk, vk, cs, pkb, vkb = transfer_keys(ctx, depth)
    rng = random.Random(42 + depth)
    rows = valid_rows(rng, batch, depth)
    rs = cport.frs([rng.randrange(R) for _ in range(2 * batch)])
    wit = oracle_witnesses(rows)
    exp = cport.Prover(cs, pkb).prove_batch(wit, rs)
    results = []
    for env in (dict(), dict(OG_CHUNK=3, OG_LANES=1), dict(OG_CHUNK=3, OG_LANES=2)):
        set_env(monkeypatch, **env)
        PK = ob.ProvingKey(ctx, pk)
        try:
            assert (PK.n_vars, PK.n_pub, PK.depth, PK.transfer_depth) == (cs.n_vars, 8, 0, depth)
            results.append(PK.prove_transfer(*pack(rows), rs))
        finally:
            PK.close()
    set_env(monkeypatch)
    nv = cs.n_vars
    for proofs, pub in results:
        assert proofs == exp
        assert pub == b"".join(wit[32 * nv * i + 32:32 * nv * i + 32 * 9] for i in range(batch))
    proofs, pub = results[0]
    assert all(proofs_verify(vk, proofs, pub, batch))
    bad = bytearray(pub[:256]); bad[32] ^= 1          # another public amount
    assert not ob.verify(vk, bytes(bad), proofs[:256])


@pytest.mark.gpu
def test_prove_transfer_dev_matches_host_entry_point(ctx):
    import torch
    pk = transfer_keys(ctx, 2)[0]
    rng = random.Random(43)
    batch = 4
    rows = valid_rows(rng, batch, 2)
    rs = cport.frs([rng.randrange(R) for _ in range(2 * batch)])
    p = pack(rows)
    PK = ob.ProvingKey(ctx, pk)
    try:
        proofs, pub = PK.prove_transfer(*p, rs)
        bits = struct.pack(f"<{2 * batch}I", *p[7])
        dev = lambda b: torch.frombuffer(bytearray(b), dtype=torch.uint8).to("cuda")
        d_in = [dev(x) for x in p[:7] + (bits,) + p[8:] + (rs,)]
        d_pr = torch.zeros(256 * batch, dtype=torch.uint8, device="cuda")
        d_pub = torch.zeros(256 * batch, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        rc = api.lib().og_groth16_prove_transfer_dev(ctx._h, PK._h, *[api._ptr(t) for t in d_in[:11]], batch, api._ptr(d_in[11]),
                                                     api._ptr(d_pr), api._ptr(d_pub))
        assert rc == 0
        ctx.sync()
        assert bytes(d_pr.cpu().numpy()) == proofs and bytes(d_pub.cpu().numpy()) == pub
    finally:
        PK.close()


@pytest.mark.gpu
def test_transfer_golden_proof(ctx):
    g = GOLD
    pk, vk = ob.setup_transfer(ctx, g["depth"], *[int(x) for x in g["toxic"]])
    v = g["vk"]
    assert vk[12:].hex() == v["alpha1"] + v["beta2"] + v["gamma2"] + v["delta2"] + v["ic"]
    rs = bn.fr_to_bytes(int(g["r"])) + bn.fr_to_bytes(int(g["s"]))
    PK = ob.ProvingKey(ctx, pk)
    try:
        proofs, pub = PK.prove_transfer(*pack([golden_row(g)]), rs)
    finally:
        PK.close()
    assert proofs.hex() == g["proof"]
    assert cport.unfr(pub) == [int(x) for x in g["public"]]
    assert ob.verify(vk, pub, proofs)


@pytest.mark.gpu
def test_bad_rows_fail_verification_alone(ctx):
    """Wrong-root and equal-nullifier rows are proved like any other; their proofs fail, the rest of the batch verifies."""
    pk, vk = transfer_keys(ctx, 2)[:2]
    rng = random.Random(44)
    rows = valid_rows(rng, 8, 2)
    rows[2]["root"] = (rows[2]["root"] + 1) % R
    r = rows[5]
    tree = mimc7.MerkleTree(2)
    notes = [(77, 1, 10), (77, 2, 20)]
    for n, s, a in notes:
        tree.insert(mimc7.multi_hash([n, s, r["token"], a]))
    r["ins"] = [(n, s, a, tree.path(i)[0], sum(b << l for l, b in enumerate(tree.path(i)[1]))) for i, (n, s, a) in enumerate(notes)]
    r["root"] = tree.root()
    rs = cport.frs([rng.randrange(R) for _ in range(16)])
    PK = ob.ProvingKey(ctx, pk)
    try:
        proofs, pub = PK.prove_transfer(*pack(rows), rs)
    finally:
        PK.close()
    assert proofs_verify(vk, proofs, pub, 8) == [i not in (2, 5) for i in range(8)]


def _generic_key(ctx, n_vars, n_pub, rng):
    cs = wc.R1CS(n_vars, n_pub)
    for j in range(n_vars - 1):
        cs.add({j: 1}, {j: 1}, {j + 1: 1})
    return ob.setup_r1cs(ctx, cs.n_vars, cs.n_pub, cs.csr("A"), cs.csr("B"), cs.csr("C"), *[rng.randrange(1, R) for _ in range(5)])[0]


@pytest.mark.gpu
def test_transfer_and_other_provers_refuse_each_others_keys(ctx):
    import torch
    d_buf = torch.zeros(1 << 16, dtype=torch.uint8, device="cuda")
    d = api._ptr(d_buf)      # every device argument of the _dev entry points
    rng = random.Random(45)
    pk_t = transfer_keys(ctx, 2)[0]
    rows = random_rows(rng, 2, 2)
    p = pack(rows)
    rs = cport.frs([rng.randrange(R) for _ in range(4)])
    tw = [rng.randrange(1, R) for _ in range(5)]
    nv2 = tc.Layout(2).n_vars
    others = [ob.setup_withdraw(ctx, 2, *tw)[0], ob.setup_deposit(ctx, *tw)[0], _generic_key(ctx, nv2, 8, rng),
              _generic_key(ctx, nv2, 7, rng)]
    bits = (api.C.c_uint32 * 4)(*p[7])
    for pk in others:
        PK = ob.ProvingKey(ctx, pk)
        try:
            with pytest.raises(ob.OwshenB200Error) as e:
                PK.prove_transfer(*p, rs)
            assert e.value.code == api.OG_E_INVALID
            args = list(p[:7]) + [bits] + list(p[8:])
            for b in (2, 0):      # the key is wrong whatever the batch
                rc = api.lib().og_groth16_prove_transfer(ctx._h, PK._h, *[api._ptr(x) for x in args], b, rs,
                                                         api.C.create_string_buffer(512), None)
                assert rc == api.OG_E_INVALID, b
                assert api.lib().og_groth16_prove_transfer_dev(ctx._h, PK._h, *[d] * 11, b, d, d, None) == api.OG_E_INVALID, b
        finally:
            PK.close()
    PK = ob.ProvingKey(ctx, pk_t)
    try:
        nul, sec, rec = (cport.frs([rng.randrange(R) for _ in range(2)]) for _ in range(3))
        for b in (2, 0):
            rc = api.lib().og_groth16_prove_withdraw(ctx._h, PK._h, nul, sec, rec, bytes(128), (api.C.c_uint32 * 2)(0, 0), b, rs,
                                                     api.C.create_string_buffer(512), None)
            assert rc == api.OG_E_INVALID, b
            assert api.lib().og_groth16_prove_withdraw_dev(ctx._h, PK._h, d, d, d, d, d, b, d, d, None) == api.OG_E_INVALID, b
        with pytest.raises(ob.OwshenB200Error) as e:
            PK.prove_deposit(nul, sec, rec, rs)
        assert e.value.code == api.OG_E_INVALID
        assert len(PK.prove_transfer(*p, rs)[0]) == 512          # the context is still usable
    finally:
        PK.close()


@pytest.mark.gpu
def test_deposit_transfer_withdraw_through_one_tree(ctx):
    """A value deposit (two dummy inputs), its notes inserted into a depth-32 tree, a private transfer spending them, and a
    withdrawal with change spending one transfer output; each proof verifies against the root of its moment."""
    pk, vk = transfer_keys(ctx, 32)[:2]
    rng = random.Random(46)
    tree = ob.MerkleTree(ctx, 32)
    tree.insert_batch([rng.randrange(R) for _ in range(3)])
    token = rng.randrange(1 << 160)
    PK = ob.ProvingKey(ctx, pk)
    leaf = lambda n, s, a: mimc7.multi_hash([n, s, token, a])
    as_int = lambda b: int.from_bytes(b, "little")

    def prove_one(r):
        rs = cport.frs([rng.randrange(R) for _ in range(2)])
        proofs, pub = PK.prove_transfer(*pack([r]), rs)
        assert ob.verify(vk, pub, proofs)
        return cport.unfr(pub)

    def spend(notes):
        ins = []
        for (n, s, a), idx in notes:
            sib, bits = tree.paths([idx])
            ins.append((n, s, a, cport.unfr(sib), bits[0]))
        return ins

    try:
        # deposit 1000 + 500 of the token: dummy inputs of value 0, proved against the current root
        dummy = [(rng.randrange(R), rng.randrange(R), 0, [0] * 32, 0) for _ in range(2)]
        d_out = [(rng.randrange(R), rng.randrange(R), 1000), (rng.randrange(R), rng.randrange(R), 500)]
        pub = prove_one(row(as_int(tree.root()), token, rng.randrange(1 << 160), dummy, d_out))
        assert pub[1] == 1500 and pub[6:8] == [leaf(*n) for n in d_out]
        idx = tree.insert_batch([pub[6], pub[7]])
        # private transfer: public amount 0
        t_out = [(rng.randrange(R), rng.randrange(R), 1200), (rng.randrange(R), rng.randrange(R), 300)]
        pub = prove_one(row(as_int(tree.root()), token, 0, spend(zip(d_out, idx)), t_out))
        assert pub[0] == as_int(tree.root()) and pub[1] == 0
        assert pub[4:6] == [mimc7.multi_hash([n[0]], key=1) for n in d_out]
        tree.insert(rng.randrange(R))
        idx = tree.insert_batch([pub[6], pub[7]])
        # withdraw 700 of the 1200 note to a recipient, 500 back as change; the second input is a dummy
        w_out = [(rng.randrange(R), rng.randrange(R), 500), (rng.randrange(R), rng.randrange(R), 0)]
        dummy_in = (rng.randrange(R), rng.randrange(R), 0, [0] * 32, 0)
        recipient = rng.randrange(1 << 160)
        pub = prove_one(row(as_int(tree.root()), token, recipient, spend([(t_out[0], idx[0])]) + [dummy_in], w_out))
        assert pub[0] == as_int(tree.root()) and pub[1] == R - 700 and pub[3] == recipient
    finally:
        PK.close()


@pytest.mark.gpu
def test_prover_plan(ctx, monkeypatch):
    set_env(monkeypatch)
    pk_w = withdraw_keys32(ctx)[0]
    pk_d = ob.setup_deposit(ctx, *[3, 5, 7, 11, 13])[0]
    for pk in (pk_w, pk_d):
        PK = ob.ProvingKey(ctx, pk)
        try:
            plan = PK.prover_plan(4096)
            assert plan["chunk"] == 1024 and plan["lanes"] == 2 and 0 < plan["scratch_bytes_per_lane"] <= LANE_BUDGET
            assert PK.prover_plan(1000) == dict(chunk=1000, lanes=1, scratch_bytes_per_lane=PK.prover_plan(1000)["scratch_bytes_per_lane"])
        finally:
            PK.close()
    PK = ob.ProvingKey(ctx, transfer_keys(ctx, 32)[0])
    try:
        plan = PK.prover_plan(4096)
        one = PK.prover_plan(1)
        assert 1 <= plan["chunk"] < 1024 and plan["lanes"] == 2
        assert plan["chunk"] == LANE_BUDGET // one["scratch_bytes_per_lane"]
        assert plan["scratch_bytes_per_lane"] <= LANE_BUDGET
        assert 2 * plan["scratch_bytes_per_lane"] < 80 * 10 ** 9
        assert PK.prover_plan(0) == dict(chunk=0, lanes=0, scratch_bytes_per_lane=0)
        set_env(monkeypatch, OG_CHUNK=3)
        assert PK.prover_plan(10)["chunk"] == 3 and PK.prover_plan(10)["lanes"] == 2
        set_env(monkeypatch, OG_CHUNK=3, OG_LANES=1)
        assert PK.prover_plan(10)["lanes"] == 1
        set_env(monkeypatch, OG_CHUNK=1500)          # above the default, within the 32-bit offset limit
        assert PK.prover_plan(100000)["chunk"] == 1500
    finally:
        set_env(monkeypatch)
        PK.close()


@pytest.mark.gpu
def test_transfer_batch_above_default_chunk(monkeypatch):
    """chunk + 1 depth-32 transfers at default settings run as two chunks on two lanes and match the oracle."""
    import torch
    set_env(monkeypatch)
    c = ob.Context(0)          # its own scratch: the session context keeps what earlier tests grew
    try:
        pk, vk, cs, pkb, vkb = transfer_keys(c, 32)
        PK = ob.ProvingKey(c, pk)
        try:
            chunk = PK.prover_plan(1 << 20)["chunk"]
            batch = chunk + 1
            plan = PK.prover_plan(batch)
            assert plan["lanes"] == 2
            need = 2 * plan["scratch_bytes_per_lane"] * 9 // 8 + 32 * batch * (cs.n_vars + 2) * 9 // 8 + 4 * GIB
            free = torch.cuda.mem_get_info()[0]
            if free < need:
                pytest.skip(f"needs ~{need / GIB:.1f} GiB of free device memory for {batch} depth-32 transfers on two lanes, "
                            f"{free / GIB:.1f} GiB free")
            rng = random.Random(47)
            rows = valid_rows(rng, 2, 32)
            rows = [rows[0]] + random_rows(rng, batch - 2, 32) + [rows[1]]
            rs = cport.frs([rng.randrange(R) for _ in range(2 * batch)])
            proofs, pub = PK.prove_transfer(*pack(rows), rs)
        finally:
            PK.close()
    finally:
        c.close()
    prover = cport.Prover(cs, pkb)
    for i in (0, batch - 1):
        wit = cport.frs(spec_witness(rows[i]))
        assert proofs[256 * i:256 * i + 256] == prover.prove_batch(wit, rs[64 * i:64 * i + 64]), i
        assert ob.verify(vk, pub[256 * i:256 * i + 256], proofs[256 * i:256 * i + 256]), i
