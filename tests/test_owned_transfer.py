"""Spend-key notes and the owned transfer statement (oracle/owned_circuit.py == csrc/withdraw_circuit.hpp:
OwnedTransferBuilder): the spec, its soundness mutations and the theft it closes, the R1CS export, the GPU hashes, witness,
setup and batched prover against the oracle, owned note delivery, and a depth-32 deposit -> delivery -> transfer -> withdrawal
chain through one tree."""
import hashlib
import json
import os
import random
import struct

import pytest

import owshen_b200 as ob
from owshen_b200 import api, formats
from oracle import bn254 as bn
from oracle import cport, mimc7
from oracle import groth16 as g16
from oracle import notes as N
from oracle import owned_circuit as oc
from oracle import transfer_circuit as tc
from oracle import withdraw_circuit as wc
from tests.helpers import pk_blob, vk_blob

R = bn.R
U64 = (1 << 64) - 1
OG_E_ENCODING = -2             # include/owshen_b200.h: a non-canonical field element
GOLD = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "owned_vectors.json")))
STATEMENTS = ("withdraw", "deposit", "transfer", "association", "exclusion", "labeled", "labeled_association", "owned_transfer")
_PROVERS = (("withdraw", 5), ("deposit", 3), ("transfer", 11), ("association", 7), ("exclusion", 9), ("labeled", 15),
            ("labeled_association", 13), ("owned_transfer", 11))
fr = lambda xs: b"".join(x.to_bytes(32, "little") for x in xs)
words = lambda b, k: [b[k * i:k * i + k] for i in range(len(b) // k)]
word_of = lambda bits: sum(b << l for l, b in enumerate(bits))


# ---- rows: one owned transfer's inputs as ints ------------------------------------------------------------------------------
def row(root, token, recipient, ins, outs):
    """ins: two (spend_key, blinding, amount, siblings, path_bits); outs: two (owner, blinding, amount)."""
    return dict(root=root, token=token, recipient=recipient, ins=ins, outs=outs)


def spec_witness(r):
    return oc.witness(r["root"], r["token"], r["recipient"], r["ins"], r["outs"])


def opened(tree, i):
    sibs, bits = tree.path(i)
    return sibs, word_of(bits)


def valid_rows(rng, batch, depth, amounts=None, token=None, first=1):
    """Rows whose input notes are leaves of one tree (a tree per row when the batch's notes do not fit in one), so every row
    satisfies the statement.  amounts: per row (in0, in1, out0, out1), default random; `first` other leaves go in first."""
    per_row = 2 * batch + first > 1 << depth
    tree, pending = None, []
    for k in range(batch):
        if tree is None or per_row:
            tree = mimc7.MerkleTree(depth)
            for _ in range(first):
                tree.insert(rng.randrange(R))
        tok = rng.randrange(R) if token is None else token
        a = amounts[k] if amounts else [rng.randrange(1 << 64) for _ in range(4)]
        notes = [(rng.randrange(R), rng.randrange(R), a[i]) for i in range(2)]
        idx = [tree.insert(oc.commitment(oc.spend_public_key(s), b, tok, am)) for s, b, am in notes]
        outs = [(oc.spend_public_key(rng.randrange(R)), rng.randrange(R), a[2 + j]) for j in range(2)]
        pending.append((tree, idx, notes, tok, outs))
    rows = []
    for tree, idx, notes, tok, outs in pending:
        ins = [(s, b, am) + opened(tree, i) for (s, b, am), i in zip(notes, idx)]
        rows.append(row(tree.root(), tok, rng.randrange(1 << 160), ins, outs))
    return rows


def random_rows(rng, batch, depth):
    """Rows of uniformly random inputs (their witnesses do not satisfy the statement: the witness kernel does not care)."""
    return [row(rng.randrange(R), rng.randrange(R), rng.randrange(R),
                [(rng.randrange(R), rng.randrange(R), rng.randrange(1 << 64), [rng.randrange(R) for _ in range(depth)],
                  rng.randrange(1 << 32)) for _ in range(2)],
                [(rng.randrange(R), rng.randrange(R), rng.randrange(1 << 64)) for _ in range(2)]) for _ in range(batch)]


def pack(rows):
    """The eleven input buffers of og_owned_transfer_witness / og_groth16_prove_owned_transfer."""
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
    for k in ("OG_CHUNK", "OG_LANES"):
        if env.get(k) is None:
            monkeypatch.delenv(k, raising=False)
        else:
            monkeypatch.setenv(k, str(env[k]))


def failing(cs, w):
    """Indices of the constraints w does not satisfy."""
    ev = wc.lc_eval
    return [k for k, (a, b, c) in enumerate(zip(cs.A, cs.B, cs.C)) if ev(a, w) * ev(b, w) % R != ev(c, w)]


# ---- CPU: the spec -------------------------------------------------------------------------------------------------------
def test_owned_transfer_sizes():
    for depth in (1, 2, 32):
        L = oc.Layout(depth)
        P = L.perm
        assert (L.n_vars, L.n_constraints) == (283 + 24 * P + depth * (4 * P + 8), 273 + 24 * P + depth * (4 * P + 6))
    expect = {32: (55867, 55793, 16), 2: (11947, 11933, 14), 1: (10483, 10471, 14)}
    for depth, (nv, nc, log_m) in expect.items():
        cs = oc.build_r1cs(depth)
        assert (cs.n_vars, cs.n_constraints, cs.n_pub) == (nv, nc, 8), depth
        assert g16.domain_log(cs.n_constraints, cs.n_pub) == log_m, depth
        assert ob.owned_transfer_r1cs_info(depth) == dict(n_constraints=nc, n_vars=nv, n_pub=8, log_m=log_m), depth
    for bad in (0, 33):
        with pytest.raises(ob.OwshenB200Error):
            ob.owned_transfer_r1cs_info(bad)


def test_eight_statement_shapes_are_distinct():
    """The prover recognises a key by (n_pub, n_vars, n_constraints): no two (statement, depth) pairs of the eight share one,
    and ProvingKey's shape lookup by (n_vars, n_pub) never takes an owned transfer key for a transfer key or back."""
    seen = {}
    for stmt in STATEMENTS:
        for d in (range(1, 33) if stmt != "deposit" else (0,)):
            i = api._statement_r1cs_info(stmt, d)
            shape = (i["n_pub"], i["n_vars"], i["n_constraints"])
            assert shape not in seen, (stmt, d, seen.get(shape))
            assert (shape[0], shape[1]) not in {(s[0], s[1]) for s in seen}, (stmt, d)
            seen[shape] = (stmt, d)
    assert sum(1 for s in seen if s[0] == 8) == 64            # n_pub = 8: the transfer and owned transfer statements


def test_owned_transfer_r1cs_export_matches_spec():
    for depth in (1, 2, 32):
        cs = oc.build_r1cs(depth)
        for m in "ABC":
            assert ob.owned_transfer_r1cs_export(depth, m) == cs.csr(m), (depth, m)


@pytest.fixture(scope="module")
def cs2():
    return oc.build_r1cs(2)


def test_owned_witnesses_satisfy(cs2):
    rng = random.Random(300)
    cases = {"deposit": (0, 0, 40, 2), "transfer": (5, 7, 9, 3), "withdrawal with change": (100, 23, 80, 0),
             "zero": (0, 0, 0, 0), "max": (U64, U64, U64, U64)}
    for name, a in cases.items():
        r = valid_rows(rng, 1, 2, [a])[0]
        if name == "deposit":    # two dummy inputs: no real path, proved against whatever the current root is
            r["ins"] = [(s, b, 0, [rng.randrange(R), rng.randrange(R)], rng.randrange(4)) for s, b, _, _, _ in r["ins"]]
        w = spec_witness(r)
        assert cs2.is_satisfied(w), name
        assert w[oc.V_PUB_AMOUNT] == (a[2] + a[3] - a[0] - a[1]) % R, name
    w = spec_witness(valid_rows(rng, 1, 2, [(100, 23, 80, 0)])[0])
    assert w[oc.V_PUB_AMOUNT] == R - 43
    # leaf indices 0 and 2^depth - 1, at depths 2 and 3
    for depth, cs in ((2, cs2), (3, oc.build_r1cs(3))):
        r = valid_rows(rng, 1, depth, [(3, 4, 5, 2)], first=0)[0]
        tree = mimc7.MerkleTree(depth)
        (s0, b0, a0, _, _), (s1, b1, a1, _, _) = r["ins"]
        tree.insert(oc.commitment(oc.spend_public_key(s0), b0, r["token"], a0))
        for _ in range((1 << depth) - 2):
            tree.insert(rng.randrange(R))
        last = tree.insert(oc.commitment(oc.spend_public_key(s1), b1, r["token"], a1))
        assert last == (1 << depth) - 1
        r = dict(r, root=tree.root(), ins=[(s0, b0, a0) + opened(tree, 0), (s1, b1, a1) + opened(tree, last)])
        w = spec_witness(r)
        assert cs.is_satisfied(w), depth
        cm1 = oc.commitment(oc.spend_public_key(s1), b1, r["token"], a1)
        assert w[oc.V_NF[1]] == oc.nullifier(s1, cm1, (1 << depth) - 1)


def test_owned_note_identities():
    rng = random.Random(301)
    r = valid_rows(rng, 1, 2)[0]
    w = spec_witness(r)
    L = oc.Layout(2)
    for j, (o, b, a) in enumerate(r["outs"]):
        assert w[oc.V_OUT_CM[j]] == mimc7.multi_hash([o, b, r["token"], a], key=4) == w[L.out(j)["cm_out"]]
    for i, (s, b, a, sibs, bits) in enumerate(r["ins"]):
        P = mimc7.multi_hash([s], key=3)
        cm = mimc7.multi_hash([P, b, r["token"], a], key=4)
        assert w[L.inp(i)["cm_out"]] == cm
        assert w[oc.V_NF[i]] == mimc7.multi_hash([s, cm, bits], key=5)
        assert mimc7.merkle_path_nodes(cm, sibs, [(bits >> l) & 1 for l in range(2)])[-1] == r["root"]
    # the same note at two leaves: two different nullifiers, both spendable in one transfer
    tree = mimc7.MerkleTree(2)
    s, b = rng.randrange(R), rng.randrange(R)
    cm = oc.commitment(oc.spend_public_key(s), b, 9, 5)
    i0, i1 = tree.insert(cm), tree.insert(cm)
    w = spec_witness(row(tree.root(), 9, 1, [(s, b, 5) + opened(tree, i0), (s, b, 5) + opened(tree, i1)], [(1, 2, 10), (3, 4, 0)]))
    assert w[oc.V_NF[0]] != w[oc.V_NF[1]] and oc.build_r1cs(2).is_satisfied(w)


def test_owned_mutations_fail_named_rows(cs2):
    rng = random.Random(302)
    L = oc.Layout(2)
    base = valid_rows(rng, 1, 2, [(6, 9, 2, 13)])[0]
    assert cs2.is_satisfied(spec_witness(base))
    # a wrong spend key: its owner, commitment and path are consistent but reach another root; only the root row fails
    r = dict(base, ins=[((base["ins"][0][0] + 1) % R,) + base["ins"][0][1:], base["ins"][1]])
    assert failing(cs2, spec_witness(r)) == [L.row_root[0]]
    # a tampered nullifier
    w = spec_witness(base)
    w[oc.V_NF[1]] = (w[oc.V_NF[1]] + 1) % R
    w[oc.V_NF_INV] = pow((w[oc.V_NF[0]] - w[oc.V_NF[1]]) % R, R - 2, R)
    assert failing(cs2, w) == [L.row_nf[1]]
    # a tampered output commitment
    w = spec_witness(base)
    w[oc.V_OUT_CM[0]] = (w[oc.V_OUT_CM[0]] + 1) % R
    assert failing(cs2, w) == [L.row_out_cm[0]]
    # a mint through r - k: output 0's amount r - 7 balances an extra 7 in output 1, but has no 64-bit decomposition
    w = spec_witness(base)
    v0, v1 = L.out(0), L.out(1)
    w[oc.V_OUT_CM[0]] = oc._note_witness(w, v0, base["outs"][0][0], base["outs"][0][0], base["outs"][0][1], base["token"], R - 7,
                                         L.perm, 91)
    w[oc.V_OUT_CM[1]] = oc._note_witness(w, v1, base["outs"][1][0], base["outs"][1][0], base["outs"][1][1], base["token"], 13 + 7 + 2,
                                         L.perm, 91)
    for k in range(64):
        w[v0["bits"] + k] = ((R - 7) >> k) & 1
    assert failing(cs2, w) == [L.row_out_range[0]]
    # an overdraw: outputs worth more than the inputs with public amount 0 leave the balance row alone unsatisfied
    r = valid_rows(rng, 1, 2, [(6, 9, 10, 6)])[0]
    w = spec_witness(r)
    w[oc.V_PUB_AMOUNT] = 0
    assert failing(cs2, w) == [L.row_balance]
    # equal nullifiers: the same note at the same leaf twice, with any nf_diff_inv
    r = dict(base, ins=[base["ins"][0], base["ins"][0]])
    w = spec_witness(r)
    assert w[oc.V_NF[0]] == w[oc.V_NF[1]] and w[oc.V_NF_INV] == 0
    for inv in (0, 1, rng.randrange(R)):
        w[oc.V_NF_INV] = inv
        assert failing(cs2, w) == [L.row_nf_diff]
    # a nonzero input under another token: its root row fails; zero-valued inputs need no path
    r = dict(base, token=(base["token"] + 1) % R)
    assert L.row_root[0] in failing(cs2, spec_witness(r))
    r = dict(base, root=(base["root"] + 1) % R)
    r["ins"] = [(s, b, 0, sb, pb) for s, b, _, sb, pb in base["ins"]]
    r["outs"] = [(1, 2, 0), (3, 4, 0)]
    assert cs2.is_satisfied(spec_witness(r))


def test_theft_by_the_sender():
    """The gap and how the owned statement closes it, three ways."""
    rng = random.Random(303)
    token = rng.randrange(1 << 160)
    # 1. transfer notes: the sender picked the output's nullifier and secret, so after it lands in the tree they can spend it
    n, s = rng.randrange(R), rng.randrange(R)
    tree = mimc7.MerkleTree(2)
    sent = tree.insert(mimc7.multi_hash([n, s, token, 50]))
    dummy = (rng.randrange(R), rng.randrange(R), 0, [0, 0], 0)
    w = tc.witness(tree.root(), token, 1, [(n, s, 50) + opened(tree, sent), dummy], [(rng.randrange(R), 1, 50), (2, 3, 0)])
    assert tc.build_r1cs(2).is_satisfied(w)
    # 2. owned notes: the sender knows P, blinding, token, amount, the leaf and its path; every s' whose P' != P fails only the
    #    root row of its input
    cs2 = oc.build_r1cs(2)
    L = oc.Layout(2)
    s_true = rng.randrange(R)
    P, b = oc.spend_public_key(s_true), rng.randrange(R)
    tree = mimc7.MerkleTree(2)
    i = tree.insert(oc.commitment(P, b, token, 50))
    dummy = (rng.randrange(R), rng.randrange(R), 0, [0, 0], 0)
    outs = [(oc.spend_public_key(rng.randrange(R)), 1, 50), (2, 3, 0)]
    for s_guess in [0, 1, P, b, R - 1] + [rng.randrange(R) for _ in range(5)]:
        assert oc.spend_public_key(s_guess) != P
        w = oc.witness(tree.root(), token, 1, [(s_guess, b, 50) + opened(tree, i), dummy], outs)
        assert failing(cs2, w) == [L.row_root[0]], s_guess
    assert cs2.is_satisfied(oc.witness(tree.root(), token, 1, [(s_true, b, 50) + opened(tree, i), dummy], outs))
    # 3. an owned leaf opened as a transfer note with nullifier = P and secret = blinding: key 4 is not key 0
    w = tc.witness(tree.root(), token, 1, [(P, b, 50) + opened(tree, i), dummy], [(rng.randrange(R), 1, 50), (2, 3, 0)])
    assert not tc.build_r1cs(2).is_satisfied(w)
    assert oc.commitment(P, b, token, 50) != mimc7.multi_hash([P, b, token, 50])


def golden_row(g):
    ins = [(int(n["spend_key"]), int(n["blinding"]), int(n["amount"]), [int(x) for x in n["siblings"]], int(n["path_bits"]))
           for n in g["inputs"]]
    outs = [(int(n["owner"]), int(n["blinding"]), int(n["amount"])) for n in g["outputs"]]
    return row(int(g["root"]), int(g["token"]), int(g["recipient"]), ins, outs)


def test_owned_golden_proof_reproduced_by_c_port():
    g = GOLD
    cs = oc.build_r1cs(g["depth"])
    pkb, vkb = cport.setup_bytes(cs, *[int(x) for x in g["toxic"]])
    assert hashlib.sha256(pkb["a"] + pkb["b1"] + pkb["b2"] + pkb["l"] + pkb["h"]).hexdigest() == g["pk_queries_sha256"]
    w = spec_witness(golden_row(g))
    assert cs.is_satisfied(w)
    wit = cport.frs(w)
    assert hashlib.sha256(wit).hexdigest() == g["witness_sha256"]
    assert cport.unfr(wit[32:32 * 9]) == [int(x) for x in g["public"]]
    assert cport.Prover(cs, pkb).prove(wit, int(g["r"]), int(g["s"])).hex() == g["proof"]
    assert ob.verify(vk_blob(vkb, 8), wit[32:32 * 9], bytes.fromhex(g["proof"]))


def test_owned_note_spec_and_envelope():
    """Owned records are the records of the four words; the owner check; the shielded-transfer envelope carries them."""
    rng = random.Random(304)
    v, s = rng.randrange(1, R), rng.randrange(R)
    P = oc.spend_public_key(s)
    note = (P, rng.randrange(R), rng.randrange(R), 77)
    e = rng.randrange(1, R)
    st, rec, cm = oc.encrypt_note(N.public_key(v), note, e)
    assert (st, rec) == N.encrypt(N.public_key(v), note, e)[:2] and cm == oc.commitment(*note)
    assert oc.scan_notes([v], [P], [rec], [cm]) == ([0], [fr(note)])
    assert oc.scan_notes([v], [P + 1], [rec], [cm])[0] == [N.NOT_OWNED]          # another spend key
    assert N.scan([v], [rec], [cm])[0] == [N.NOT_OWNED]                            # a key-0 scan does not see it
    proof, pub = bytes(rng.randrange(256) for _ in range(256)), fr([rng.randrange(R) for _ in range(8)])
    recs = rec + oc.encrypt_note(N.public_key(v), note, e + 1)[1]
    assert formats.shielded_transfer_from_rlp(formats.shielded_transfer_to_rlp(proof, pub, recs)) == (proof, pub, recs)


# ---- GPU -----------------------------------------------------------------------------------------------------------------
_KEYS = {}


def keys(ctx, depth):
    """(pk, vk, r1cs, oracle pk bytes, oracle vk bytes) of the depth-`depth` owned transfer statement, made once per process."""
    if depth not in _KEYS:
        rng = random.Random(310 + depth)
        tw = [rng.randrange(1, R) for _ in range(5)]
        pk, vk = ob.setup_owned_transfer(ctx, depth, *tw)
        cs = oc.build_r1cs(depth)
        pkb, vkb = cport.setup_bytes(cs, *tw)
        _KEYS[depth] = (pk, vk, cs, pkb, vkb)
    return _KEYS[depth]


def proofs_verify(vk, proofs, pub, batch):
    return [ob.verify(vk, pub[256 * i:256 * i + 256], proofs[256 * i:256 * i + 256]) for i in range(batch)]


@pytest.mark.gpu
def test_owned_hashes_match_oracle(ctx):
    rng = random.Random(305)
    for n in (1, 63, 64, 65, 200):
        ks = [rng.randrange(R) for _ in range(n)] if n > 2 else [0]
        ks[-1] = R - 1
        assert ctx.owned_public_keys(fr(ks)) == fr([oc.spend_public_key(k) for k in ks]), n
        notes = [(rng.randrange(R), rng.randrange(R), rng.randrange(R), [0, U64, rng.randrange(1 << 64)][i % 3]) for i in range(n)]
        got = ctx.owned_commitments(*[fr([m[k] for m in notes]) for k in range(3)], [m[3] for m in notes])
        assert got == fr([oc.commitment(*m) for m in notes]), n
        idx = [[0, (1 << 32) - 1, rng.randrange(1 << 32)][i % 3] for i in range(n)]
        cms = [rng.randrange(R) for _ in range(n)]
        assert ctx.owned_nullifiers(fr(ks), fr(cms), idx) == fr([oc.nullifier(k, c, i) for k, c, i in zip(ks, cms, idx)]), n
    bad = R.to_bytes(32, "little")
    for call in (lambda: ctx.owned_public_keys(bad), lambda: ctx.owned_commitments(bad, fr([1]), fr([1]), [1]),
                 lambda: ctx.owned_commitments(fr([1]), fr([1]), bad, [1]), lambda: ctx.owned_nullifiers(fr([1]), bad, [0]),
                 lambda: ctx.owned_nullifiers(bad, fr([1]), [0])):
        with pytest.raises(ob.OwshenB200Error) as e:
            call()
        assert e.value.code == OG_E_ENCODING
    with pytest.raises(ValueError):
        ctx.owned_nullifiers(fr([1]), fr([1]), [1 << 32])


@pytest.mark.gpu
def test_owned_transfer_witness_matches_oracle(ctx):
    rng = random.Random(306)
    for depth in (2, 32):
        rows = random_rows(rng, 37 if depth == 2 else 5, depth) + valid_rows(rng, 3, depth)
        assert ctx.owned_transfer_witness(depth, *pack(rows)) == oracle_witnesses(rows), depth
    # edge values: amounts 0, 1, 2^64 - 1; field inputs 0 and r - 1; one note twice (nullifier difference 0, inverse 0)
    rows = []
    for a in (0, 1, U64):
        for x in (0, R - 1):
            rows.append(row(x, x, x, [(x, x, a, [x, x], 3), ((x + 1) % R, x, a, [x, x], 0)], [(x, x, a), (x, x, a)]))
    rows.append(row(5, 6, 7, [(9, 1, 2, [3, 4], 1), (9, 1, 2, [3, 4], 1)], [(1, 1, 1), (2, 2, 4)]))
    got = ctx.owned_transfer_witness(2, *pack(rows))
    assert got == oracle_witnesses(rows)
    nv = oc.Layout(2).n_vars
    assert got[32 * nv * (len(rows) - 1) + 32 * oc.V_NF_INV:][:32] == bytes(32)
    for k in (0, 1, 2, 3, 4, 6, 8, 9):          # a field input >= r
        p = list(pack(rows[:1]))
        p[k] = R.to_bytes(32, "little") + p[k][32:]
        with pytest.raises(ob.OwshenB200Error) as e:
            ctx.owned_transfer_witness(2, *p)
        assert e.value.code == OG_E_ENCODING, k


@pytest.mark.gpu
def test_setup_owned_transfer_matches_oracle(ctx):
    for depth in (2, 32):
        pk, vk, cs, pkb, vkb = keys(ctx, depth)
        assert pk == pk_blob(cs, pkb, 0), depth
        assert vk == vk_blob(vkb, 8), depth


@pytest.mark.gpu
def test_owned_transfer_key_from_ceremony(ctx):
    rng = random.Random(307)
    t, a, b, d = (rng.randrange(1, R) for _ in range(4))
    acc0 = ob.ptau_new(ctx, 14)                           # the depth-2 owned transfer domain is 2^14
    acc1, rec = ob.ptau_contribute(ctx, acc0, [t, a, b], [rng.randrange(1, R) for _ in range(3)])
    assert ob.ptau_verify(ctx, acc0, acc1, rec)
    pk0, vk0 = ob.ptau_prepare_owned_transfer(ctx, acc1, 2)
    assert (pk0, vk0) == ob.setup_owned_transfer(ctx, 2, t, a, b, 1, 1)
    pk, vk, rec2 = ob.phase2_contribute(ctx, pk0, vk0, d, rng.randrange(1, R))
    assert ob.phase2_verify(ctx, pk0, vk0, pk, vk, rec2)
    assert (pk, vk) == ob.setup_owned_transfer(ctx, 2, t, a, b, 1, d)
    PK = ob.ProvingKey(ctx, pk)
    try:
        assert (PK.owned_transfer_depth, PK.transfer_depth) == (2, None)
    finally:
        PK.close()


@pytest.mark.gpu
@pytest.mark.parametrize("depth,batch", [(2, 40), (32, 3)])
def test_prove_owned_transfer_matches_oracle(ctx, monkeypatch, depth, batch):
    """Default settings, then chunks below the batch on one and two lanes: all byte for byte the oracle C prover's."""
    pk, vk, cs, pkb, vkb = keys(ctx, depth)
    rng = random.Random(320 + depth)
    rows = valid_rows(rng, batch, depth)
    rs = cport.frs([rng.randrange(R) for _ in range(2 * batch)])
    wit = oracle_witnesses(rows)
    exp = cport.Prover(cs, pkb).prove_batch(wit, rs)
    results = []
    chunk = 3 if depth == 2 else 2
    for env in (dict(), dict(OG_CHUNK=chunk, OG_LANES=1), dict(OG_CHUNK=chunk, OG_LANES=2)):
        set_env(monkeypatch, **env)
        PK = ob.ProvingKey(ctx, pk)
        try:
            assert (PK.n_vars, PK.n_pub, PK.depth, PK.owned_transfer_depth, PK.transfer_depth) == (cs.n_vars, 8, 0, depth, None)
            results.append(PK.prove_owned_transfer(*pack(rows), rs))
        finally:
            PK.close()
    set_env(monkeypatch)
    nv = cs.n_vars
    for proofs, pub in results:
        assert proofs == exp
        assert pub == b"".join(wit[32 * nv * i + 32:32 * nv * i + 32 * 9] for i in range(batch))
    proofs, pub = results[0]
    assert all(proofs_verify(vk, proofs, pub, batch))
    bad = bytearray(pub[:256]); bad[32 * 4] ^= 1          # another nullifier
    assert not ob.verify(vk, bytes(bad), proofs[:256])


@pytest.mark.gpu
def test_prove_owned_transfer_dev_matches_host_entry_point(ctx):
    import torch
    pk = keys(ctx, 2)[0]
    rng = random.Random(308)
    batch = 4
    rows = valid_rows(rng, batch, 2)
    rs = cport.frs([rng.randrange(R) for _ in range(2 * batch)])
    p = pack(rows)
    PK = ob.ProvingKey(ctx, pk)
    try:
        proofs, pub = PK.prove_owned_transfer(*p, rs)
        bits = struct.pack(f"<{2 * batch}I", *p[7])
        dev = lambda b: torch.frombuffer(bytearray(b), dtype=torch.uint8).to("cuda")
        d_in = [dev(x) for x in p[:7] + (bits,) + p[8:] + (rs,)]
        d_pr = torch.zeros(256 * batch, dtype=torch.uint8, device="cuda")
        d_pub = torch.zeros(256 * batch, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        rc = api.lib().og_groth16_prove_owned_transfer_dev(ctx._h, PK._h, *[api._ptr(t) for t in d_in[:11]], batch,
                                                           api._ptr(d_in[11]), api._ptr(d_pr), api._ptr(d_pub))
        assert rc == 0
        ctx.sync()
        assert bytes(d_pr.cpu().numpy()) == proofs and bytes(d_pub.cpu().numpy()) == pub
    finally:
        PK.close()


@pytest.mark.gpu
def test_owned_golden_proof(ctx):
    g = GOLD
    pk, vk = ob.setup_owned_transfer(ctx, g["depth"], *[int(x) for x in g["toxic"]])
    v = g["vk"]
    assert vk[12:].hex() == v["alpha1"] + v["beta2"] + v["gamma2"] + v["delta2"] + v["ic"]
    rs = bn.fr_to_bytes(int(g["r"])) + bn.fr_to_bytes(int(g["s"]))
    PK = ob.ProvingKey(ctx, pk)
    try:
        proofs, pub = PK.prove_owned_transfer(*pack([golden_row(g)]), rs)
    finally:
        PK.close()
    assert proofs.hex() == g["proof"]
    assert cport.unfr(pub) == [int(x) for x in g["public"]]
    assert ob.verify(vk, pub, proofs)


@pytest.mark.gpu
def test_eight_provers_refuse_each_others_keys(ctx):
    import torch
    d_buf = torch.zeros(1 << 16, dtype=torch.uint8, device="cuda")
    d = api._ptr(d_buf)                                   # every device argument of the _dev entry points
    h = bytes(1 << 16)                                    # every host input of the host entry points
    rng = random.Random(309)
    tw = [rng.randrange(1, R) for _ in range(5)]
    all_keys = {"withdraw": ob.setup_withdraw(ctx, 2, *tw)[0], "deposit": ob.setup_deposit(ctx, *tw)[0],
                "transfer": ob.setup_transfer(ctx, 2, *tw)[0], "association": ob.setup_association(ctx, 2, *tw)[0],
                "exclusion": ob.setup_exclusion(ctx, 2, *tw)[0], "labeled": ob.setup_labeled(ctx, 2, *tw)[0],
                "labeled_association": ob.setup_labeled_association(ctx, 2, *tw)[0], "owned_transfer": keys(ctx, 2)[0]}
    for owner, pk in all_keys.items():
        PK = ob.ProvingKey(ctx, pk)
        try:
            for stmt, n_in in _PROVERS:
                if stmt == owner:
                    continue
                for b in (2, 0):
                    host = getattr(api.lib(), f"og_groth16_prove_{stmt}")
                    rc = host(ctx._h, PK._h, *[h] * n_in, b, h, api.C.create_string_buffer(512), None)
                    assert rc == api.OG_E_INVALID, (owner, stmt, b)
                    dev = getattr(api.lib(), f"og_groth16_prove_{stmt}_dev")
                    assert dev(ctx._h, PK._h, *[d] * n_in, b, d, d, None) == api.OG_E_INVALID, (owner, stmt, b)
            if owner != "owned_transfer":
                with pytest.raises(ob.OwshenB200Error):
                    PK.prove_owned_transfer(*pack(valid_rows(rng, 1, 2)), bytes(64))
        finally:
            PK.close()
    PK = ob.ProvingKey(ctx, all_keys["owned_transfer"])
    try:
        rows = valid_rows(rng, 2, 2)
        assert len(PK.prove_owned_transfer(*pack(rows), cport.frs([rng.randrange(R) for _ in range(4)]))[0]) == 512
    finally:
        PK.close()


def owned_encrypt(ctx, pks, notes, es, owned=True):
    enc = ctx.owned_note_encrypt if owned else ctx.note_encrypt
    return enc(fr([p[0] for p in pks]), bytes(p[1] for p in pks), *[fr([m[k] for m in notes]) for k in range(3)],
               [m[3] for m in notes], fr(es))


@pytest.mark.gpu
def test_owned_note_encrypt_and_scan_match_oracle(ctx):
    import torch
    from tests.golden.gen_note_golden import non_decompressing_x, set_word
    rng = random.Random(311)
    view = [rng.randrange(1, R) for _ in range(3)]
    spend = [rng.randrange(R) for _ in range(3)]
    P = [oc.spend_public_key(s) for s in spend]
    addr = [N.public_key(v) for v in view]
    n = 130
    pks = [addr[i % 3] for i in range(n)]
    pks[5] = (non_decompressing_x(), 0)                     # refused key
    es = [rng.randrange(1, R) for _ in range(n)]
    es[6] = 0                                               # refused ephemeral
    notes = []
    for i in range(n):
        owner = P[i % 3] if i % 5 != 1 else (P[(i + 1) % 3] if i % 2 else rng.randrange(R))   # to v_k, but another spend key
        notes.append((owner, rng.randrange(R), rng.randrange(R), [0, U64, rng.randrange(1 << 64)][i % 3]))
    rec, cm, st = owned_encrypt(ctx, pks, notes, es)
    spec = [oc.encrypt_note(p, m, e) for p, m, e in zip(pks, notes, es)]
    assert list(st) == [x[0] for x in spec] and {1, 2, 3} <= set(st)
    assert rec == b"".join(x[1] for x in spec) and cm == fr([x[2] for x in spec])
    # the same four words through og_note_encrypt: byte-identical records, key-0 commitments
    rec0, cm0, st0 = owned_encrypt(ctx, pks, notes, es, owned=False)
    assert (rec0, st0) == (rec, st) and cm0 == fr([N.encrypt(p, m, e)[2] for p, m, e in zip(pks, notes, es)])
    # malformed and tampered records behave as before
    recs, cms = words(rec, 160), [int.from_bytes(c, "little") for c in words(cm, 32)]
    recs[7] = set_word(recs[7], 0, non_decompressing_x())
    recs[8] = set_word(recs[8], 2, R + 5)
    cms[9] = R + 1
    recs[10] = set_word(recs[10], 3, int.from_bytes(recs[10][96:128], "little") ^ 4)
    expect = oc.scan_notes(view, P, recs, cms)
    got_o, got_p = ctx.owned_note_scan(fr(view), fr(P), b"".join(recs), fr(cms))
    assert got_o == expect[0] and words(got_p, 128) == expect[1]
    assert got_o[7] == got_o[8] == got_o[9] == N.MALFORMED and got_o[10] == N.NOT_OWNED
    ok = [i for i in range(n) if st[i] == 1 and i not in (7, 8, 9, 10)]
    assert all(got_o[i] == (i % 3 if i % 5 != 1 else N.NOT_OWNED) for i in ok)
    # key-0 and key-4 records never cross between the two scans
    assert set(ctx.note_scan(fr(view), b"".join(recs), fr(cms))[0]) <= {N.NOT_OWNED, N.MALFORMED}
    recs0 = words(rec0, 160)
    assert set(ctx.owned_note_scan(fr(view), fr(P), rec0, cm0)[0]) <= {N.NOT_OWNED, N.MALFORMED}
    assert ctx.note_scan(fr(view), rec0, cm0)[0] == N.scan(view, recs0, [int.from_bytes(c, "little") for c in words(cm0, 32)])[0]
    # the _dev variants
    dev = torch.device("cuda", ctx.device)
    u8 = lambda b: torch.frombuffer(bytearray(b), dtype=torch.uint8).to(dev)
    ins = [u8(fr([p[0] for p in pks])), u8(bytes(p[1] for p in pks))] + [u8(fr([m[k] for m in notes])) for k in range(3)]
    ins += [u8(struct.pack(f"<{n}Q", *[m[3] for m in notes])), u8(fr(es))]
    d_rec, d_cm, d_st = (torch.zeros(k * n, dtype=torch.uint8, device=dev) for k in (160, 32, 1))
    ctx.owned_note_encrypt_dev(*ins, n, d_rec, d_cm, d_st)
    ctx.sync()
    assert (bytes(d_rec.cpu().numpy()), bytes(d_cm.cpu().numpy()), bytes(d_st.cpu().numpy())) == (rec, cm, st)
    d_owner = torch.zeros(n, dtype=torch.int32, device=dev)
    d_plain = torch.zeros(128 * n, dtype=torch.uint8, device=dev)
    ctx.owned_note_scan_dev(fr(view), fr(P), u8(b"".join(recs)), u8(fr(cms)), n, d_owner, d_plain)
    ctx.sync()
    assert [x & 0xFFFFFFFF for x in d_owner.cpu().tolist()] == got_o and bytes(d_plain.cpu().numpy()) == got_p
    # argument errors: a non-canonical spend public key, unequal key lists
    with pytest.raises(ob.OwshenB200Error) as e:
        ctx.owned_note_scan(fr(view), fr(P[:2]) + R.to_bytes(32, "little"), rec, cm)
    assert e.value.code == OG_E_ENCODING
    with pytest.raises(ValueError):
        ctx.owned_note_scan(fr(view), fr(P[:2]), rec, cm)
    assert ctx.owned_note_scan(b"", b"", rec, cm)[0] == [N.MALFORMED if i in (5, 6) else N.NOT_OWNED for i in range(n)]


@pytest.mark.gpu
def test_owned_deposit_delivery_transfer_withdraw_chain(ctx):
    """Through one depth-32 tree with plain notes between the owned ones: an owned deposit (two dummy inputs) is appended and
    delivered to a recipient, who scans, computes its nullifier and transfers to a third party with change; the third party
    withdraws.  The original sender's attempt to spend the delivered note gives a proof that fails verification, and a
    second spend of one note reproduces its nullifier."""
    pk, vk = keys(ctx, 32)[:2]
    rng = random.Random(312)
    tree = ob.MerkleTree(ctx, 32)
    tree.insert_batch([rng.randrange(R) for _ in range(3)])
    token = rng.randrange(1 << 160)
    PK = ob.ProvingKey(ctx, pk)
    as_int = lambda b: int.from_bytes(b, "little")
    fr1 = lambda x: x.to_bytes(32, "little")

    def prove(root, ins, outs, recipient=0):
        r = row(root, token, recipient, ins, outs)
        proofs, pub = PK.prove_owned_transfer(*pack([r]), cport.frs([rng.randrange(R) for _ in range(2)]))
        assert pub == cport.frs(spec_witness(r)[1:9])
        return proofs, pub

    def spend_in(s, b, a, index):
        sib, bits = tree.paths([index])
        return (s, b, a, cport.unfr(sib), bits[0])

    try:
        # wallets: (view key, spending key) each; the sender has one too
        (va, sa), (vb, sb), (vs, ss) = [(rng.randrange(1, R), rng.randrange(R)) for _ in range(3)]
        Pa, Pb = (as_int(x) for x in words(ctx.owned_public_keys(fr([sa, sb])), 32))
        assert (Pa, Pb) == (oc.spend_public_key(sa), oc.spend_public_key(sb))
        # 1. the sender deposits 100 to A: two dummy inputs against the current root
        dummies = [(rng.randrange(R), rng.randrange(R), 0, [0] * 32, 0), (rng.randrange(R), rng.randrange(R), 0, [0] * 32, 1)]
        blind = rng.randrange(R)
        outs = [(Pa, blind, 100), (oc.spend_public_key(ss), rng.randrange(R), 0)]
        proofs, pub = prove(as_int(tree.root()), dummies, outs)
        assert ob.verify(vk, pub, proofs) and as_int(pub[32:64]) == 100
        cm_a = as_int(pub[32 * 6:32 * 7])
        assert fr1(cm_a) == ctx.owned_commitments(fr1(Pa), fr1(blind), fr1(token), [100])
        # 2. appended between plain leaves, and delivered to A's view key
        idx_a = tree.insert(cm_a)
        tree.insert_batch([rng.randrange(R) for _ in range(2)])
        rec, cm, st = owned_encrypt(ctx, [N.public_key(va)], [(Pa, blind, token, 100)], [rng.randrange(1, R)])
        assert st == b"\x01" and as_int(cm) == cm_a
        msg = formats.shielded_transfer_to_rlp(proofs, pub, rec + rec)
        assert formats.shielded_transfer_from_rlp(msg)[2][:160] == rec
        # 3. A scans (with a foreign wallet's key first), finds the note and its nullifier
        owners, plain = ctx.owned_note_scan(fr([vs, va]), fr([oc.spend_public_key(ss), Pa]), rec, cm)
        assert owners == [1]
        P_, b_, t_, a_ = (as_int(x) for x in words(plain, 32))
        assert (P_, b_, t_, a_) == (Pa, blind, token, 100)
        nf_a = as_int(ctx.owned_nullifiers(fr1(sa), cm, [idx_a]))
        root = as_int(tree.root())
        # the sender, who knows everything about the note but sa, cannot make a verifying spend
        for guess in (ss, Pa, blind):
            proofs, pub = prove(root, [spend_in(guess, blind, 100, idx_a), dummies[1]], [(Pa, 1, 100), (Pa, 2, 0)])
            assert not ob.verify(vk, pub, proofs), guess
        # A transfers 60 to B with 40 change to A, spending the note; a second spend reproduces the nullifier
        b_change, b_out = rng.randrange(R), rng.randrange(R)
        ins = [spend_in(sa, blind, 100, idx_a), dummies[1]]
        proofs, pub = prove(root, ins, [(Pb, b_out, 60), (Pa, b_change, 40)])
        assert ob.verify(vk, pub, proofs) and as_int(pub[32:64]) == 0 and as_int(pub[32 * 4:32 * 5]) == nf_a
        proofs2, pub2 = prove(root, ins, [(Pb, b_out, 60), (Pa, b_change, 40)])
        assert ob.verify(vk, pub2, proofs2) and pub2[32 * 4:32 * 5] == pub[32 * 4:32 * 5]
        cm_b, cm_change = as_int(pub[32 * 6:32 * 7]), as_int(pub[32 * 7:32 * 8])
        idx_b = tree.insert(cm_b)
        tree.insert(rng.randrange(R))
        tree.insert(cm_change)
        # 4. B withdraws 25 of its 60 to a recipient, keeping 35
        root = as_int(tree.root())
        recipient = rng.randrange(1 << 160)
        proofs, pub = prove(root, [spend_in(sb, b_out, 60, idx_b), dummies[0]], [(Pb, rng.randrange(R), 35), (Pb, 0, 0)], recipient)
        assert ob.verify(vk, pub, proofs)
        assert as_int(pub[32:64]) == R - 25 and as_int(pub[32 * 3:32 * 4]) == recipient
        assert as_int(pub[32 * 4:32 * 5]) == as_int(ctx.owned_nullifiers(fr1(sb), fr1(cm_b), [idx_b]))
    finally:
        PK.close()
