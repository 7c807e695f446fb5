"""Owned labeled notes and the owned labeled transfer statement (oracle/owned_labeled_circuit.py == csrc/withdraw_circuit.hpp:
OwnedLabeledTransferBuilder): the spec, its soundness mutations and domain separation, the R1CS export, the GPU hashes,
witness, setup and batched prover against the oracle, owned labeled note delivery, and a depth-32 chain of deposits,
approval, a transfer, delivery and a withdrawal through one pool tree and one ApprovedLabels set."""
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
from oracle import labeled_association_circuit as lac
from oracle import labeled_circuit as lc
from oracle import notes as N
from oracle import owned_circuit as oc
from oracle import owned_labeled_circuit as olc
from oracle import transfer_circuit as tc
from oracle import withdraw_circuit as wc
from tests.helpers import pk_blob, vk_blob

R = bn.R
U64 = (1 << 64) - 1
OG_E_ENCODING = -2             # include/owshen_b200.h: a non-canonical field element
GOLD = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "owned_labeled_vectors.json")))
STATEMENTS = ("withdraw", "deposit", "transfer", "association", "exclusion", "labeled", "labeled_association", "owned_transfer",
              "owned_labeled_transfer")
_PROVERS = (("withdraw", 5), ("deposit", 3), ("transfer", 11), ("association", 7), ("exclusion", 9), ("labeled", 15),
            ("labeled_association", 13), ("owned_transfer", 11), ("owned_labeled_transfer", 15))
fr = lambda xs: b"".join(x.to_bytes(32, "little") for x in xs)
words = lambda b, k: [b[k * i:k * i + k] for i in range(len(b) // k)]
word_of = lambda bits: sum(b << l for l, b in enumerate(bits))


# ---- rows: one owned labeled transfer's inputs as ints -----------------------------------------------------------------------
def row(root, token, withdrawn, recipient, label, ins, outs, asibs, abits):
    """ins: two (spend_key, blinding, amount, siblings, path_bits); outs: two (owner, blinding, amount); asibs/abits: the
    association path of label + 1."""
    return dict(root=root, token=token, withdrawn=withdrawn, recipient=recipient, label=label, ins=ins, outs=outs, asibs=asibs,
                abits=abits)


def spec_witness(r):
    return olc.witness(r["root"], r["token"], r["withdrawn"], r["recipient"], r["label"], r["ins"], r["outs"], r["asibs"], r["abits"])


def opened(tree, i):
    sibs, bits = tree.path(i)
    return sibs, word_of(bits)


def valid_rows(rng, batch, depth, amounts=None, label=None, first=1):
    """Rows whose input notes are leaves of one pool tree per row under the row's label, which an approved-label tree holds,
    so every row satisfies the statement.  amounts: per row (in0, in1, out0, out1, withdrawn), default random balanced."""
    rows = []
    for k in range(batch):
        la = rng.randrange(min(1 << depth, 1 << 32)) if label is None else label
        tree = mimc7.MerkleTree(depth)
        for _ in range(first):
            tree.insert(rng.randrange(R))
        tok = rng.randrange(R)
        if amounts:
            a = amounts[k]
        else:
            i0, i1 = rng.randrange(1 << 63), rng.randrange(1 << 63)
            wd = rng.randrange(i0 + 1)
            o0 = rng.randrange(i0 + i1 - wd + 1)
            a = (i0, i1, o0, i0 + i1 - wd - o0, wd)
        notes = [(rng.randrange(R), rng.randrange(R), a[i]) for i in range(2)]
        idx = [tree.insert(olc.note_leaf(olc.spend_public_key(s), b, tok, am, la)) for s, b, am in notes]
        outs = [(olc.spend_public_key(rng.randrange(R)), rng.randrange(R), a[2 + j]) for j in range(2)]
        approved = lac.ApprovedTree(depth, [la] + ([la ^ 1] if depth > 1 else []))
        asibs, abits = approved.path(la)
        ins = [(s, b, am) + opened(tree, i) for (s, b, am), i in zip(notes, idx)]
        rows.append(row(tree.root(), tok, a[4], rng.randrange(1 << 160), la, ins, outs, asibs, word_of(abits)))
    return rows


def random_rows(rng, batch, depth):
    """Rows of uniformly random inputs (their witnesses do not satisfy the statement: the witness kernel does not care)."""
    return [row(rng.randrange(R), rng.randrange(R), rng.randrange(1 << 64), rng.randrange(R), rng.randrange(1 << 32),
                [(rng.randrange(R), rng.randrange(R), rng.randrange(1 << 64), [rng.randrange(R) for _ in range(depth)],
                  rng.randrange(1 << 32)) for _ in range(2)],
                [(rng.randrange(R), rng.randrange(R), rng.randrange(1 << 64)) for _ in range(2)],
                [rng.randrange(R) for _ in range(depth)], rng.randrange(1 << 32)) for _ in range(batch)]


def pack(rows):
    """The fifteen input buffers of og_owned_labeled_transfer_witness / og_groth16_prove_owned_labeled_transfer."""
    f = cport.frs
    u64 = lambda xs: struct.pack(f"<{len(xs)}Q", *xs)
    return (f([r["root"] for r in rows]), f([r["token"] for r in rows]), f([r["recipient"] for r in rows]),
            u64([r["withdrawn"] for r in rows]), [r["label"] for r in rows],
            f([n[0] for r in rows for n in r["ins"]]), f([n[1] for r in rows for n in r["ins"]]),
            u64([n[2] for r in rows for n in r["ins"]]), f([s for r in rows for n in r["ins"] for s in n[3]]),
            [n[4] for r in rows for n in r["ins"]],
            f([n[0] for r in rows for n in r["outs"]]), f([n[1] for r in rows for n in r["outs"]]),
            u64([n[2] for r in rows for n in r["outs"]]), f([s for r in rows for s in r["asibs"]]), [r["abits"] for r in rows])


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
def test_owned_labeled_transfer_sizes():
    for depth in (1, 2, 32):
        L = olc.Layout(depth)
        P = L.perm
        assert (L.n_vars, L.n_constraints) == (386 + 32 * P + depth * (6 * P + 12), 377 + 32 * P + depth * (6 * P + 9))
    expect = {32: (82306, 82201, 17), 2: (16426, 16411, 15), 1: (14230, 14218, 14)}
    for depth, (nv, nc, log_m) in expect.items():
        cs = olc.build_r1cs(depth)
        assert (cs.n_vars, cs.n_constraints, cs.n_pub) == (nv, nc, 9), depth
        assert g16.domain_log(cs.n_constraints, cs.n_pub) == log_m, depth
        assert ob.owned_labeled_transfer_r1cs_info(depth) == dict(n_constraints=nc, n_vars=nv, n_pub=9, log_m=log_m), depth
    for bad in (0, 33):
        with pytest.raises(ob.OwshenB200Error):
            ob.owned_labeled_transfer_r1cs_info(bad)


def test_nine_statement_shapes_are_distinct():
    """The prover recognises a key by (n_pub, n_vars, n_constraints) and ProvingKey by (n_vars, n_pub): no two (statement,
    depth) pairs of the nine share either."""
    seen = {}
    for stmt in STATEMENTS:
        for d in (range(1, 33) if stmt != "deposit" else (0,)):
            i = api._statement_r1cs_info(stmt, d)
            shape = (i["n_pub"], i["n_vars"], i["n_constraints"])
            assert shape not in seen, (stmt, d, seen.get(shape))
            assert (shape[0], shape[1]) not in {(s[0], s[1]) for s in seen}, (stmt, d)
            seen[shape] = (stmt, d)
    assert [s[0] for s in seen].count(9) == 32                # n_pub = 9: this statement alone


def test_owned_labeled_transfer_r1cs_export_matches_spec():
    for depth in (1, 2, 32):
        cs = olc.build_r1cs(depth)
        for m in "ABC":
            assert ob.owned_labeled_transfer_r1cs_export(depth, m) == cs.csr(m), (depth, m)


@pytest.fixture(scope="module")
def cs2():
    return olc.build_r1cs(2)


def _with_ins(r, ins, root=None):
    return dict(r, ins=ins, root=r["root"] if root is None else root)


def test_owned_labeled_witnesses_satisfy(cs2):
    rng = random.Random(400)
    cases = {"private transfer": (5, 7, 9, 3, 0), "withdrawal with change": (100, 23, 80, 0, 43),
             "full withdrawal": (100, 23, 0, 0, 123), "zero": (0, 0, 0, 0, 0), "max": (U64, 0, U64, 0, 0),
             "max withdrawn": (U64, 0, 0, 0, U64)}
    for name, a in cases.items():
        w = spec_witness(valid_rows(rng, 1, 2, [a])[0])
        assert cs2.is_satisfied(w), name
        assert w[olc.V_WITHDRAWN] == a[4], name
    # a dummy input in either position: no real path, any label
    for pos in (0, 1):
        r = valid_rows(rng, 1, 2, [(30, 30, 25, 5, 0) if pos else (30, 30, 5, 25, 0)])[0]
        ins = list(r["ins"])
        ins[pos] = (rng.randrange(R), rng.randrange(R), 0, [rng.randrange(R), rng.randrange(R)], rng.randrange(4))
        assert cs2.is_satisfied(spec_witness(_with_ins(r, ins))), pos
    # labels 0 and 2^depth - 1, leaf indices 0 and 2^depth - 1, at depths 2 and 3
    for depth, cs in ((2, cs2), (3, olc.build_r1cs(3))):
        for la in (0, (1 << depth) - 1):
            r = valid_rows(rng, 1, depth, [(3, 4, 5, 1, 1)], label=la, first=0)[0]
            tree = mimc7.MerkleTree(depth)
            (s0, b0, a0, _, _), (s1, b1, a1, _, _) = r["ins"]
            tree.insert(olc.note_leaf(olc.spend_public_key(s0), b0, r["token"], a0, la))
            for _ in range((1 << depth) - 2):
                tree.insert(rng.randrange(R))
            last = tree.insert(olc.note_leaf(olc.spend_public_key(s1), b1, r["token"], a1, la))
            assert last == (1 << depth) - 1
            r = _with_ins(r, [(s0, b0, a0) + opened(tree, 0), (s1, b1, a1) + opened(tree, last)], tree.root())
            w = spec_witness(r)
            assert cs.is_satisfied(w), (depth, la)
            lf1 = olc.note_leaf(olc.spend_public_key(s1), b1, r["token"], a1, la)
            assert w[olc.V_NF[1]] == olc.nullifier(s1, lf1, (1 << depth) - 1)
    # one note at two leaves: two different nullifiers, both spendable in one transfer
    r = valid_rows(rng, 1, 2, [(5, 5, 10, 0, 0)])[0]
    tree = mimc7.MerkleTree(2)
    s, b = rng.randrange(R), rng.randrange(R)
    lf = olc.note_leaf(olc.spend_public_key(s), b, r["token"], 5, r["label"])
    i0, i1 = tree.insert(lf), tree.insert(lf)
    w = spec_witness(_with_ins(r, [(s, b, 5) + opened(tree, i0), (s, b, 5) + opened(tree, i1)], tree.root()))
    assert w[olc.V_NF[0]] != w[olc.V_NF[1]] and cs2.is_satisfied(w)


def test_owned_labeled_note_identities():
    rng = random.Random(401)
    r = valid_rows(rng, 1, 2)[0]
    w = spec_witness(r)
    L = olc.Layout(2)
    la, tok = r["label"], r["token"]
    for j, (o, b, a) in enumerate(r["outs"]):
        pre = mimc7.multi_hash([o, b], key=6)
        assert w[olc.V_OUT_CM[j]] == mimc7.multi_hash([pre, tok, a, la], key=7) == w[L.out(j)["leaf_out"]]
    for i, (s, b, a, sibs, bits) in enumerate(r["ins"]):
        lf = mimc7.multi_hash([mimc7.multi_hash([mimc7.multi_hash([s], key=3), b], key=6), tok, a, la], key=7)
        assert w[L.inp(i)["leaf_out"]] == lf
        assert w[olc.V_NF[i]] == mimc7.multi_hash([s, lf, bits], key=5) == oc.nullifier(s, lf, bits)
    assert w[olc.V_ALEAF] == la + 1


def test_owned_labeled_mutations_fail_named_rows(cs2):
    rng = random.Random(402)
    L = olc.Layout(2)
    base = valid_rows(rng, 1, 2, [(6, 9, 2, 10, 3)], label=2)[0]
    assert cs2.is_satisfied(spec_witness(base))
    # a wrong spend key: owner, leaf and path are consistent but reach another root; only the root row fails
    r = _with_ins(base, [((base["ins"][0][0] + 1) % R,) + base["ins"][0][1:], base["ins"][1]])
    assert failing(cs2, spec_witness(r)) == [L.row_root[0]]
    # two nonzero inputs of different labels: input 1 is a leaf under label 1, the transaction's label is 2
    tree = mimc7.MerkleTree(2)
    (s0, b0, a0, _, _), (s1, b1, a1, _, _) = base["ins"]
    i0 = tree.insert(olc.note_leaf(olc.spend_public_key(s0), b0, base["token"], a0, 2))
    i1 = tree.insert(olc.note_leaf(olc.spend_public_key(s1), b1, base["token"], a1, 1))
    r = _with_ins(base, [(s0, b0, a0) + opened(tree, i0), (s1, b1, a1) + opened(tree, i1)], tree.root())
    assert failing(cs2, spec_witness(r)) == [L.row_root[1]]
    # an unapproved label with another (approved) label's association path
    approved = lac.ApprovedTree(2, [1, 3])
    asibs, abits = approved.path(1)
    r = dict(base, asibs=asibs, abits=word_of(abits))
    w = spec_witness(r)
    w[olc.V_AROOT] = approved.root()
    assert failing(cs2, w) == [L.row_assoc_root]
    # label = r - 1 on an empty slot: assoc_leaf = 0 is an empty leaf of the tree, the label's range row fails (the leaves
    # and the root rows fail too: a label that is not the deposit's)
    r = dict(base, label=R - 1, asibs=approved.tree.path(2)[0], abits=word_of(approved.tree.path(2)[1]))
    w = spec_witness(r)
    assert w[olc.V_ALEAF] == 0 and w[olc.V_AROOT] == approved.root()
    assert L.row_label_range in failing(cs2, w) and L.row_assoc_root not in failing(cs2, w)
    # assoc_leaf != label + 1: the leaf of the next label, with its consistent path, fails the assoc_leaf row alone
    w = spec_witness(base)
    w[olc.V_ALEAF] = (w[olc.V_ALEAF] + 1) % R
    w[olc.V_AROOT] = olc._levels_witness(w, L, olc.ASSOC, w[olc.V_ALEAF], base["asibs"], base["abits"])
    assert failing(cs2, w) == [L.row_assoc_leaf]
    # withdrawn = r - k: outputs worth k more than the inputs, the balance holds mod r, the withdrawn range row fails
    r = valid_rows(rng, 1, 2, [(6, 9, 10, 12, 0)], label=2)[0]
    r["withdrawn"] = R - 7
    assert failing(cs2, spec_witness(r)) == [L.row_withdrawn_range]
    # an overdraw: outputs worth more than the inputs
    r = valid_rows(rng, 1, 2, [(6, 9, 10, 6, 0)], label=2)[0]
    assert failing(cs2, spec_witness(r)) == [L.row_balance]
    # the forbidden deposit: two dummy inputs and nonzero outputs
    r = valid_rows(rng, 1, 2, [(0, 0, 40, 2, 0)], label=2)[0]
    r = _with_ins(r, [(rng.randrange(R), rng.randrange(R), 0, [0, 0], 0) for _ in range(2)])
    assert failing(cs2, spec_witness(r)) == [L.row_balance]
    # a tampered nullifier
    w = spec_witness(base)
    w[olc.V_NF[1]] = (w[olc.V_NF[1]] + 1) % R
    w[olc.V_NF_INV] = pow((w[olc.V_NF[0]] - w[olc.V_NF[1]]) % R, R - 2, R)
    assert failing(cs2, w) == [L.row_nf[1]]
    # a tampered out_commitment
    w = spec_witness(base)
    w[olc.V_OUT_CM[0]] = (w[olc.V_OUT_CM[0]] + 1) % R
    assert failing(cs2, w) == [L.row_out_cm[0]]
    # equal nullifiers: the same note at the same leaf twice, with any nf_diff_inv
    r = _with_ins(base, [base["ins"][0], base["ins"][0]])
    r["outs"] = [(1, 2, 9), (3, 4, 0)]                    # 6 + 6 = 9 + 0 + withdrawn 3
    w = spec_witness(r)
    assert w[olc.V_NF[0]] == w[olc.V_NF[1]] and w[olc.V_NF_INV] == 0
    for inv in (0, 1, rng.randrange(R)):
        w[olc.V_NF_INV] = inv
        assert failing(cs2, w) == [L.row_nf_diff]


def test_domain_separation_and_the_sender():
    rng = random.Random(403)
    token, la = rng.randrange(1 << 160), 1
    s, b = rng.randrange(R), rng.randrange(R)
    P = olc.spend_public_key(s)
    pre = olc.precommitment(P, b)
    tree = mimc7.MerkleTree(2)
    tree.insert(rng.randrange(R))
    i = tree.insert(olc.leaf(pre, token, 50, la))
    sibs, bits = opened(tree, i)
    dummy = (rng.randrange(R), rng.randrange(R), 0, [0, 0], 0)
    approved = lac.ApprovedTree(2, [la])
    asibs, abits = approved.path(la)
    # an owned labeled leaf opened as an owned note (key 4), a transfer note (key 0) or a labeled note (key 2)
    w = oc.witness(tree.root(), token, 1, [(s, b, 50, sibs, bits), dummy], [(P, 1, 50), (2, 3, 0)])
    assert not oc.build_r1cs(2).is_satisfied(w)
    w = tc.witness(tree.root(), token, 1, [(P, b, 50, sibs, bits), dummy], [(1, 1, 50), (2, 3, 0)])
    assert not tc.build_r1cs(2).is_satisfied(w)
    bl = [(bits >> l) & 1 for l in range(2)]
    w = lac.witness(P, b, 1, token, 0, 50, la, sibs, bl, 1, 2, asibs, abits)
    w[lac.V_ROOT] = tree.root()                           # the labeled witness derives root; the pool's is what counts
    assert not lac.build_r1cs(2).is_satisfied(w)
    # owned (key 4) and labeled (key 2) leaves are not spendable here
    for foreign in (oc.commitment(P, b, token, 50), lc.leaf(lc.precommitment(P, b), token, 50, la)):
        t = mimc7.MerkleTree(2)
        j = t.insert(foreign)
        w = olc.witness(t.root(), token, 0, 1, la, [(s, b, 50) + opened(t, j), dummy], [(P, 1, 50), (P, 2, 0)], asibs, word_of(abits))
        assert not olc.build_r1cs(2).is_satisfied(w)
    # the sender knows P, blinding, the precommitment, the leaf and its path but not s: every guess fails the root row only
    cs2 = olc.build_r1cs(2)
    L = olc.Layout(2)
    for guess in [0, 1, P, b, pre, R - 1] + [rng.randrange(R) for _ in range(4)]:
        w = olc.witness(tree.root(), token, 0, 1, la, [(guess, b, 50, sibs, bits), dummy], [(P, 1, 50), (P, 2, 0)], asibs,
                        word_of(abits))
        assert failing(cs2, w) == [L.row_root[0]], guess
    assert cs2.is_satisfied(olc.witness(tree.root(), token, 0, 1, la, [(s, b, 50, sibs, bits), dummy], [(P, 1, 50), (P, 2, 0)],
                                        asibs, word_of(abits)))


def golden_row(g):
    ins = [(int(n["spend_key"]), int(n["blinding"]), int(n["amount"]), [int(x) for x in n["siblings"]], int(n["path_bits"]))
           for n in g["inputs"]]
    outs = [(int(n["owner"]), int(n["blinding"]), int(n["amount"])) for n in g["outputs"]]
    return row(int(g["root"]), int(g["token"]), int(g["withdrawn"]), int(g["recipient"]), int(g["label"]), ins, outs,
               [int(x) for x in g["assoc_siblings"]], int(g["assoc_path_bits"]))


def test_owned_labeled_golden_proof_reproduced_by_c_port():
    g = GOLD
    cs = olc.build_r1cs(g["depth"])
    pkb, vkb = cport.setup_bytes(cs, *[int(x) for x in g["toxic"]])
    assert hashlib.sha256(pkb["a"] + pkb["b1"] + pkb["b2"] + pkb["l"] + pkb["h"]).hexdigest() == g["pk_queries_sha256"]
    w = spec_witness(golden_row(g))
    assert cs.is_satisfied(w)
    wit = cport.frs(w)
    assert hashlib.sha256(wit).hexdigest() == g["witness_sha256"]
    assert cport.unfr(wit[32:32 * 10]) == [int(x) for x in g["public"]]
    assert cport.Prover(cs, pkb).prove(wit, int(g["r"]), int(g["s"])).hex() == g["proof"]
    assert ob.verify(vk_blob(vkb, 9), wit[32:32 * 10], bytes.fromhex(g["proof"]))


def test_owned_labeled_note_spec_and_envelope():
    """Records of the four words with the label packed into word 3; the owner and range checks; the envelope."""
    rng = random.Random(404)
    v, s = rng.randrange(1, R), rng.randrange(R)
    P = olc.spend_public_key(s)
    note = (P, rng.randrange(R), rng.randrange(R), U64, (1 << 32) - 1)
    e = rng.randrange(1, R)
    st, rec, cm = olc.encrypt_note(N.public_key(v), note, e)
    assert st == N.ENC_OK and cm == olc.note_leaf(*note)
    assert olc.scan_notes([v], [P], [rec], [cm]) == ([0], [fr(olc.pack_words(note))])
    assert olc.scan_notes([v], [P + 1], [rec], [cm])[0] == [N.NOT_OWNED]          # another spend key
    assert oc.scan_notes([v], [P], [rec], [cm])[0] == [N.NOT_OWNED]                # not an owned (key-4) note
    assert N.scan([v], [rec], [cm])[0] == [N.NOT_OWNED]                            # nor a transfer note
    # an owned note's record is not owned in this scan
    onote = (P, rng.randrange(R), rng.randrange(R), 5)
    _, orec, ocm = oc.encrypt_note(N.public_key(v), onote, e)
    assert olc.scan_notes([v], [P], [orec], [ocm])[0] == [N.NOT_OWNED]
    assert olc.unpack_words((1, 2, 3, 1 << 96)) is None
    proof, pub = bytes(rng.randrange(256) for _ in range(256)), fr([rng.randrange(R) for _ in range(9)])
    recs = rec + olc.encrypt_note(N.public_key(v), note, e + 1)[1]
    msg = formats.shielded_labeled_transfer_to_rlp(proof, pub, recs)
    assert formats.shielded_labeled_transfer_from_rlp(msg) == (proof, pub, recs)
    bad = [formats.shielded_transfer_to_rlp(proof, pub[:256], recs), formats.rlp_encode(["shielded-labeled-transfer", proof]),
           formats.rlp_encode(["shielded-labeled-transfer", proof] + words(pub, 32) + [recs[:160], recs[160:319]]),
           formats.rlp_encode(["shielded-labeled-transfer", proof[:255]] + words(pub, 32) + words(recs, 160)),
           formats.rlp_encode(["shielded-transfer", proof] + words(pub, 32) + words(recs, 160)), msg + b"\x00"]
    for m in bad:
        with pytest.raises(ValueError):
            formats.shielded_labeled_transfer_from_rlp(m)
    with pytest.raises(ValueError):
        formats.shielded_transfer_from_rlp(msg)
    with pytest.raises(ValueError):
        formats.shielded_labeled_transfer_to_rlp(proof, pub[:256], recs)


# ---- GPU -----------------------------------------------------------------------------------------------------------------
_KEYS = {}


def keys(ctx, depth):
    """(pk, vk, r1cs, oracle pk bytes, oracle vk bytes) of the depth-`depth` owned labeled transfer statement, once per
    process."""
    if depth not in _KEYS:
        rng = random.Random(410 + depth)
        tw = [rng.randrange(1, R) for _ in range(5)]
        pk, vk = ob.setup_owned_labeled_transfer(ctx, depth, *tw)
        cs = olc.build_r1cs(depth)
        pkb, vkb = cport.setup_bytes(cs, *tw)
        _KEYS[depth] = (pk, vk, cs, pkb, vkb)
    return _KEYS[depth]


def proofs_verify(vk, proofs, pub, batch):
    return [ob.verify(vk, pub[288 * i:288 * i + 288], proofs[256 * i:256 * i + 256]) for i in range(batch)]


@pytest.mark.gpu
def test_owned_labeled_hashes_match_oracle(ctx):
    rng = random.Random(405)
    for n in (1, 63, 64, 65, 200):
        owners = [rng.randrange(R) for _ in range(n)]
        owners[-1] = R - 1
        bl = [rng.randrange(R) for _ in range(n)]
        pre = ctx.owned_labeled_precommitments(fr(owners), fr(bl))
        assert pre == fr([olc.precommitment(o, b) for o, b in zip(owners, bl)]), n
        toks = [rng.randrange(R) for _ in range(n)]
        ams = [[0, U64, rng.randrange(1 << 64)][i % 3] for i in range(n)]
        las = [[0, (1 << 32) - 1, rng.randrange(1 << 32)][i % 3] for i in range(n)]
        leaves = ctx.owned_labeled_leaves(pre, fr(toks), ams, las)
        spec = [olc.leaf(p, t, a, la) for p, t, a, la in zip(cport.unfr(pre), toks, ams, las)]
        assert leaves == fr(spec), n
        ks, idx = [rng.randrange(R) for _ in range(n)], [rng.randrange(1 << 32) for _ in range(n)]
        assert ctx.owned_nullifiers(fr(ks), leaves, idx) == fr([olc.nullifier(k, c, i) for k, c, i in zip(ks, spec, idx)]), n
    bad = R.to_bytes(32, "little")
    for call in (lambda: ctx.owned_labeled_precommitments(bad, fr([1])), lambda: ctx.owned_labeled_precommitments(fr([1]), bad),
                 lambda: ctx.owned_labeled_leaves(bad, fr([1]), [1], [1]), lambda: ctx.owned_labeled_leaves(fr([1]), bad, [1], [1])):
        with pytest.raises(ob.OwshenB200Error) as e:
            call()
        assert e.value.code == OG_E_ENCODING
    with pytest.raises(ValueError):
        ctx.owned_labeled_leaves(fr([1]), fr([1]), [1], [1 << 32])


@pytest.mark.gpu
def test_owned_labeled_transfer_witness_matches_oracle(ctx):
    rng = random.Random(406)
    for depth in (2, 32):
        rows = random_rows(rng, 37 if depth == 2 else 5, depth) + valid_rows(rng, 3, depth)
        assert ctx.owned_labeled_transfer_witness(depth, *pack(rows)) == oracle_witnesses(rows), depth
    # edge values: amounts and withdrawn 0 and 2^64 - 1, labels 0 and 2^32 - 1, field inputs 0 and r - 1, one note twice
    rows = []
    for a, la in ((0, 0), (1, (1 << 32) - 1), (U64, 7)):
        for x in (0, R - 1):
            rows.append(row(x, x, a, x, la, [(x, x, a, [x, x], 3), ((x + 1) % R, x, a, [x, x], 0)], [(x, x, a), (x, x, a)],
                            [x, x], 2))
    rows.append(row(5, 6, 0, 7, 1, [(9, 1, 2, [3, 4], 1), (9, 1, 2, [3, 4], 1)], [(1, 1, 1), (2, 2, 3)], [3, 4], 1))
    got = ctx.owned_labeled_transfer_witness(2, *pack(rows))
    assert got == oracle_witnesses(rows)
    nv = olc.Layout(2).n_vars
    assert got[32 * nv * (len(rows) - 1) + 32 * olc.V_NF_INV:][:32] == bytes(32)
    for k in (0, 1, 2, 5, 6, 8, 10, 11, 13):          # a field input >= r
        p = list(pack(rows[:1]))
        p[k] = R.to_bytes(32, "little") + p[k][32:]
        with pytest.raises(ob.OwshenB200Error) as e:
            ctx.owned_labeled_transfer_witness(2, *p)
        assert e.value.code == OG_E_ENCODING, k
    # the boundary: depth 0 and 33, null pointers
    bufs = [api._u32_array(x) if isinstance(x, list) else x for x in pack(rows[:1])]
    out = api.C.create_string_buffer(32 * nv)
    for d in (0, 33):
        assert api.lib().og_owned_labeled_transfer_witness(ctx._h, d, *[api._ptr(x) for x in bufs], 1, out) == api.OG_E_INVALID, d
    for k in range(15):
        args = [api._ptr(x) for x in bufs]
        args[k] = None
        assert api.lib().og_owned_labeled_transfer_witness(ctx._h, 2, *args, 1, out) == api.OG_E_INVALID, k


@pytest.mark.gpu
def test_setup_owned_labeled_transfer_matches_oracle(ctx):
    for depth in (2, 32):
        pk, vk, cs, pkb, vkb = keys(ctx, depth)
        assert pk == pk_blob(cs, pkb, 0), depth
        assert vk == vk_blob(vkb, 9), depth


@pytest.mark.gpu
def test_owned_labeled_transfer_key_from_ceremony(ctx):
    rng = random.Random(407)
    t, a, b, d = (rng.randrange(1, R) for _ in range(4))
    acc0 = ob.ptau_new(ctx, 15)                           # the depth-2 domain is 2^15
    acc1, rec = ob.ptau_contribute(ctx, acc0, [t, a, b], [rng.randrange(1, R) for _ in range(3)])
    assert ob.ptau_verify(ctx, acc0, acc1, rec)
    pk0, vk0 = ob.ptau_prepare_owned_labeled_transfer(ctx, acc1, 2)
    assert (pk0, vk0) == ob.setup_owned_labeled_transfer(ctx, 2, t, a, b, 1, 1)
    pk, vk, rec2 = ob.phase2_contribute(ctx, pk0, vk0, d, rng.randrange(1, R))
    assert ob.phase2_verify(ctx, pk0, vk0, pk, vk, rec2)
    assert (pk, vk) == ob.setup_owned_labeled_transfer(ctx, 2, t, a, b, 1, d)
    PK = ob.ProvingKey(ctx, pk)
    try:
        assert (PK.owned_labeled_transfer_depth, PK.owned_transfer_depth) == (2, None)
    finally:
        PK.close()


@pytest.mark.gpu
@pytest.mark.parametrize("depth,batch", [(2, 40), (32, 3)])
def test_prove_owned_labeled_transfer_matches_oracle(ctx, monkeypatch, depth, batch):
    """Default settings, then chunks below the batch on one and two lanes: all byte for byte the oracle C prover's."""
    pk, vk, cs, pkb, vkb = keys(ctx, depth)
    rng = random.Random(420 + depth)
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
            assert (PK.n_vars, PK.n_pub, PK.depth, PK.owned_labeled_transfer_depth) == (cs.n_vars, 9, 0, depth)
            results.append(PK.prove_owned_labeled_transfer(*pack(rows), rs))
        finally:
            PK.close()
    set_env(monkeypatch)
    nv = cs.n_vars
    for proofs, pub in results:
        assert proofs == exp
        assert pub == b"".join(wit[32 * nv * i + 32:32 * nv * i + 32 * 10] for i in range(batch))
    proofs, pub = results[0]
    assert all(proofs_verify(vk, proofs, pub, batch))
    bad = bytearray(pub[:288]); bad[32 * 5] ^= 1          # another nullifier
    assert not ob.verify(vk, bytes(bad), proofs[:256])


@pytest.mark.gpu
def test_prove_owned_labeled_transfer_dev_matches_host_entry_point(ctx):
    import torch
    pk = keys(ctx, 2)[0]
    rng = random.Random(408)
    batch = 4
    rows = valid_rows(rng, batch, 2)
    rs = cport.frs([rng.randrange(R) for _ in range(2 * batch)])
    p = pack(rows)
    PK = ob.ProvingKey(ctx, pk)
    try:
        proofs, pub = PK.prove_owned_labeled_transfer(*p, rs)
        u32 = lambda xs: struct.pack(f"<{len(xs)}I", *xs)
        host = [u32(x) if isinstance(x, list) else x for x in p]
        dev = lambda b: torch.frombuffer(bytearray(b), dtype=torch.uint8).to("cuda")
        d_in = [dev(x) for x in host + [rs]]
        d_pr = torch.zeros(256 * batch, dtype=torch.uint8, device="cuda")
        d_pub = torch.zeros(288 * batch, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        rc = api.lib().og_groth16_prove_owned_labeled_transfer_dev(ctx._h, PK._h, *[api._ptr(t) for t in d_in[:15]], batch,
                                                                   api._ptr(d_in[15]), api._ptr(d_pr), api._ptr(d_pub))
        assert rc == 0
        ctx.sync()
        assert bytes(d_pr.cpu().numpy()) == proofs and bytes(d_pub.cpu().numpy()) == pub
    finally:
        PK.close()


@pytest.mark.gpu
def test_owned_labeled_golden_proof(ctx):
    g = GOLD
    pk, vk = ob.setup_owned_labeled_transfer(ctx, g["depth"], *[int(x) for x in g["toxic"]])
    v = g["vk"]
    assert vk[12:].hex() == v["alpha1"] + v["beta2"] + v["gamma2"] + v["delta2"] + v["ic"]
    rs = bn.fr_to_bytes(int(g["r"])) + bn.fr_to_bytes(int(g["s"]))
    PK = ob.ProvingKey(ctx, pk)
    try:
        proofs, pub = PK.prove_owned_labeled_transfer(*pack([golden_row(g)]), rs)
    finally:
        PK.close()
    assert proofs.hex() == g["proof"]
    assert cport.unfr(pub) == [int(x) for x in g["public"]]
    assert ob.verify(vk, pub, proofs)


@pytest.mark.gpu
def test_nine_provers_refuse_each_others_keys(ctx):
    import torch
    d_buf = torch.zeros(1 << 16, dtype=torch.uint8, device="cuda")
    d = api._ptr(d_buf)                                   # every device argument of the _dev entry points
    h = bytes(1 << 16)                                    # every host input of the host entry points
    rng = random.Random(409)
    tw = [rng.randrange(1, R) for _ in range(5)]
    all_keys = {"withdraw": ob.setup_withdraw(ctx, 2, *tw)[0], "deposit": ob.setup_deposit(ctx, *tw)[0],
                "transfer": ob.setup_transfer(ctx, 2, *tw)[0], "association": ob.setup_association(ctx, 2, *tw)[0],
                "exclusion": ob.setup_exclusion(ctx, 2, *tw)[0], "labeled": ob.setup_labeled(ctx, 2, *tw)[0],
                "labeled_association": ob.setup_labeled_association(ctx, 2, *tw)[0],
                "owned_transfer": ob.setup_owned_transfer(ctx, 2, *tw)[0], "owned_labeled_transfer": keys(ctx, 2)[0]}
    for owner, pk in all_keys.items():
        PK = ob.ProvingKey(ctx, pk)
        try:
            for stmt, n_in in _PROVERS:
                if stmt == owner:
                    continue
                for b in (2, 0):
                    host = getattr(api.lib(), f"og_groth16_prove_{stmt}")
                    rc = host(ctx._h, PK._h, *[h] * n_in, b, h, api.C.create_string_buffer(576), None)
                    assert rc == api.OG_E_INVALID, (owner, stmt, b)
                    dev = getattr(api.lib(), f"og_groth16_prove_{stmt}_dev")
                    assert dev(ctx._h, PK._h, *[d] * n_in, b, d, d, None) == api.OG_E_INVALID, (owner, stmt, b)
            if owner != "owned_labeled_transfer":
                with pytest.raises(ob.OwshenB200Error):
                    PK.prove_owned_labeled_transfer(*pack(valid_rows(rng, 1, 2)), bytes(64))
        finally:
            PK.close()
    PK = ob.ProvingKey(ctx, all_keys["owned_labeled_transfer"])
    try:
        rows = valid_rows(rng, 2, 2)
        assert len(PK.prove_owned_labeled_transfer(*pack(rows), cport.frs([rng.randrange(R) for _ in range(4)]))[0]) == 512
    finally:
        PK.close()


def labeled_encrypt(ctx, pks, notes, es):
    return ctx.owned_labeled_note_encrypt(fr([p[0] for p in pks]), bytes(p[1] for p in pks), *[fr([m[k] for m in notes]) for k in range(3)],
                                          [m[3] for m in notes], [m[4] for m in notes], fr(es))


@pytest.mark.gpu
def test_owned_labeled_note_encrypt_and_scan_match_oracle(ctx):
    import torch
    from tests.golden.gen_note_golden import non_decompressing_x, set_word
    rng = random.Random(411)
    view = [rng.randrange(1, R) for _ in range(3)]
    spend = [rng.randrange(R) for _ in range(3)]
    P = [olc.spend_public_key(s) for s in spend]
    addr = [N.public_key(v) for v in view]
    n = 130
    pks = [addr[i % 3] for i in range(n)]
    pks[5] = (non_decompressing_x(), 0)                     # refused key
    es = [rng.randrange(1, R) for _ in range(n)]
    es[6] = 0                                               # refused ephemeral
    notes = []
    for i in range(n):
        owner = P[i % 3] if i % 5 != 1 else (P[(i + 1) % 3] if i % 2 else rng.randrange(R))   # to v_k, but another spend key
        notes.append((owner, rng.randrange(R), rng.randrange(R), [0, U64, rng.randrange(1 << 64)][i % 3],
                      [0, (1 << 32) - 1, rng.randrange(1 << 32)][i % 3]))
    rec, cm, st = labeled_encrypt(ctx, pks, notes, es)
    spec = [olc.encrypt_note(p, m, e) for p, m, e in zip(pks, notes, es)]
    assert list(st) == [x[0] for x in spec] and {1, 2, 3} <= set(st)
    assert rec == b"".join(x[1] for x in spec) and cm == fr([x[2] for x in spec])
    recs, cms = words(rec, 160), [int.from_bytes(c, "little") for c in words(cm, 32)]
    recs[7] = set_word(recs[7], 0, non_decompressing_x())
    recs[8] = set_word(recs[8], 2, R + 5)
    cms[9] = R + 1
    recs[10] = set_word(recs[10], 3, int.from_bytes(recs[10][96:128], "little") ^ 4)
    expect = olc.scan_notes(view, P, recs, cms)
    got_o, got_p, got_a, got_l = ctx.owned_labeled_note_scan(fr(view), fr(P), b"".join(recs), fr(cms))
    assert got_o == expect[0] and words(got_p, 128) == expect[1]
    assert got_o[7] == got_o[8] == got_o[9] == N.MALFORMED and got_o[10] == N.NOT_OWNED
    ok = [i for i in range(n) if st[i] == 1 and i not in (7, 8, 9, 10)]
    assert all(got_o[i] == (i % 3 if i % 5 != 1 else N.NOT_OWNED) for i in ok)
    assert all((got_a[i], got_l[i]) == ((notes[i][3], notes[i][4]) if got_o[i] < 3 else (0, 0)) for i in range(n))
    # transfer-note and owned-note records are not owned in this scan, and this family's are not owned in theirs
    assert set(ctx.note_scan(fr(view), b"".join(recs), fr(cms))[0]) <= {N.NOT_OWNED, N.MALFORMED}
    assert set(ctx.owned_note_scan(fr(view), fr(P), b"".join(recs), fr(cms))[0]) <= {N.NOT_OWNED, N.MALFORMED}
    onotes = [(m[0], m[1], m[2], m[3]) for m in notes]
    orec, ocm, _ = ctx.owned_note_encrypt(fr([p[0] for p in pks]), bytes(p[1] for p in pks), *[fr([m[k] for m in onotes]) for k in range(3)],
                                          [m[3] for m in onotes], fr(es))
    assert set(ctx.owned_labeled_note_scan(fr(view), fr(P), orec, ocm)[0]) <= {N.NOT_OWNED, N.MALFORMED}
    trec, tcm, _ = ctx.note_encrypt(fr([p[0] for p in pks]), bytes(p[1] for p in pks), *[fr([m[k] for m in onotes]) for k in range(3)],
                                    [m[3] for m in onotes], fr(es))
    assert set(ctx.owned_labeled_note_scan(fr(view), fr(P), trec, tcm)[0]) <= {N.NOT_OWNED, N.MALFORMED}
    # the _dev variants
    dev = torch.device("cuda", ctx.device)
    u8 = lambda b: torch.frombuffer(bytearray(b), dtype=torch.uint8).to(dev)
    ins = [u8(fr([p[0] for p in pks])), u8(bytes(p[1] for p in pks))] + [u8(fr([m[k] for m in notes])) for k in range(3)]
    ins += [u8(struct.pack(f"<{n}Q", *[m[3] for m in notes])), u8(struct.pack(f"<{n}I", *[m[4] for m in notes])), u8(fr(es))]
    d_rec, d_cm, d_st = (torch.zeros(k * n, dtype=torch.uint8, device=dev) for k in (160, 32, 1))
    ctx.owned_labeled_note_encrypt_dev(*ins, n, d_rec, d_cm, d_st)
    ctx.sync()
    assert (bytes(d_rec.cpu().numpy()), bytes(d_cm.cpu().numpy()), bytes(d_st.cpu().numpy())) == (rec, cm, st)
    d_owner = torch.zeros(n, dtype=torch.int32, device=dev)
    d_plain = torch.zeros(128 * n, dtype=torch.uint8, device=dev)
    ctx.owned_labeled_note_scan_dev(fr(view), fr(P), u8(b"".join(recs)), u8(fr(cms)), n, d_owner, d_plain)
    ctx.sync()
    assert [x & 0xFFFFFFFF for x in d_owner.cpu().tolist()] == got_o and bytes(d_plain.cpu().numpy()) == got_p
    with pytest.raises(ob.OwshenB200Error) as e:
        ctx.owned_labeled_note_scan(fr(view), fr(P[:2]) + R.to_bytes(32, "little"), rec, cm)
    assert e.value.code == OG_E_ENCODING
    with pytest.raises(ValueError):
        ctx.owned_labeled_note_scan(fr(view), fr(P[:2]), rec, cm)


@pytest.mark.gpu
def test_owned_labeled_deposit_approve_transfer_withdraw_chain(ctx):
    """Through one depth-32 pool tree with plain and labeled deposits between the owned labeled ones, and one ApprovedLabels
    set: A transfers to B with change under one label, B finds the note by scanning and withdraws part of it.  A's spend of
    B's note, a second spend, a join of two deposits and an unapproved deposit all behave as the policy says, and the same
    approved root serves a labeled association withdrawal."""
    from owshen_b200 import ApprovedLabels
    pk, vk = keys(ctx, 32)[:2]
    rng = random.Random(412)
    tree = ob.MerkleTree(ctx, 32)
    tree.insert_batch([rng.randrange(R) for _ in range(3)])
    token = rng.randrange(1 << 160)
    PK = ob.ProvingKey(ctx, pk)
    as_int = lambda b: int.from_bytes(b, "little")
    fr1 = lambda x: x.to_bytes(32, "little")
    try:
        (va, sa), (vb, sb) = [(rng.randrange(1, R), rng.randrange(R)) for _ in range(2)]
        Pa, Pb = (as_int(x) for x in words(ctx.owned_public_keys(fr([sa, sb])), 32))
        # 1. owned labeled deposits between plain and labeled ones
        ba = [rng.randrange(R) for _ in range(3)]
        pre = ctx.owned_labeled_precommitments(fr([Pa] * 3), fr(ba))
        amts = [100, 70, 55]
        la = ob.deposit_owned_labeled(tree, pre[:32], fr1(token), amts[:1])
        lpre = ctx.labeled_precommitments(fr([7]), fr([8]))
        l_label = ob.deposit_labeled(tree, lpre, fr1(token), [40])
        tree.insert(rng.randrange(R))
        lb = ob.deposit_owned_labeled(tree, pre[32:], fr([token, token]), amts[1:])
        labels = la + lb
        assert labels == [3, 6, 7] and l_label == [4]
        # 2. the provider approves some deposits
        approved = ApprovedLabels(ctx, 32, [labels[0], labels[1], l_label[0]])
        aroot = as_int(approved.root())

        def spend_in(s, b, a, index):
            sib, bits = tree.paths([index])
            return (s, b, a, cport.unfr(sib), bits[0])

        def prove(label, ins, outs, withdrawn=0, recipient=0, apath=None):
            asib, abits = approved.witness([label]) if apath is None else apath
            r = row(as_int(tree.root()), token, withdrawn, recipient, label, ins, outs, cport.unfr(asib), abits[0])
            proofs, pub = PK.prove_owned_labeled_transfer(*pack([r]), cport.frs([rng.randrange(R) for _ in range(2)]))
            assert pub == cport.frs(spec_witness(r)[1:10])
            return proofs, pub

        dummy = (rng.randrange(R), rng.randrange(R), 0, [0] * 32, 0)
        # 3. A transfers 60 of deposit 3 to B with 40 change to A, under label 3
        b_out, b_ch = rng.randrange(R), rng.randrange(R)
        ins = [spend_in(sa, ba[0], 100, labels[0]), dummy]
        proofs, pub = prove(labels[0], ins, [(Pb, b_out, 60), (Pa, b_ch, 40)])
        assert ob.verify(vk, pub, proofs) and as_int(pub[32:64]) == aroot
        nf_a = as_int(pub[32 * 5:32 * 6])
        leaf_a = olc.note_leaf(Pa, ba[0], token, 100, labels[0])
        assert nf_a == as_int(ctx.owned_nullifiers(fr1(sa), fr1(leaf_a), [labels[0]]))
        # 7. a second spend repeats its nullifier
        proofs2, pub2 = prove(labels[0], ins, [(Pb, b_out, 60), (Pa, b_ch, 40)])
        assert ob.verify(vk, pub2, proofs2) and pub2[32 * 5:32 * 6] == pub[32 * 5:32 * 6]
        cm_b = as_int(pub[32 * 7:32 * 8])
        idx_b = tree.insert(cm_b)
        tree.insert(as_int(pub[32 * 8:32 * 9]))
        # 4. delivery; B's scan recovers amount and label
        addr_b = N.public_key(vb)
        rec, cm, st = ctx.owned_labeled_note_encrypt(fr1(addr_b[0]), bytes([addr_b[1]]), fr1(Pb), fr1(b_out), fr1(token), [60], [labels[0]])
        assert st == b"\x01" and as_int(cm) == cm_b
        msg = formats.shielded_labeled_transfer_to_rlp(proofs, pub, rec + rec)
        assert formats.shielded_labeled_transfer_from_rlp(msg)[2][:160] == rec
        owners, plain, amounts, lbls = ctx.owned_labeled_note_scan(fr([va, vb]), fr([Pa, Pb]), rec, cm)
        assert owners == [1] and (amounts, lbls) == ([60], [labels[0]])
        # 5. B withdraws 25 to a recipient, keeping 35
        recipient = rng.randrange(1 << 160)
        proofs, pub = prove(labels[0], [spend_in(sb, b_out, 60, idx_b), dummy], [(Pb, rng.randrange(R), 35), (Pb, 0, 0)], 25,
                            recipient)
        assert ob.verify(vk, pub, proofs) and as_int(pub[32 * 3:32 * 4]) == 25 and as_int(pub[32 * 4:32 * 5]) == recipient
        # 6. A's attempt to spend B's note fails verification
        for guess in (sa, Pb, b_out):
            proofs, pub = prove(labels[0], [spend_in(guess, b_out, 60, idx_b), dummy], [(Pa, 1, 60), (Pa, 2, 0)])
            assert not ob.verify(vk, pub, proofs), guess
        # 8. joining notes of two deposits (labels 3 and 6) fails, under either label
        for label in labels[:2]:
            proofs, pub = prove(label, [spend_in(sa, ba[0], 100, labels[0]), spend_in(sa, ba[1], 70, labels[1])],
                                [(Pa, 1, 170), (Pa, 2, 0)])
            assert not ob.verify(vk, pub, proofs), label
        # 9. an unapproved deposit has no witness, fails with a neighbour's path, and succeeds after approve()
        with pytest.raises(ValueError):
            approved.witness([labels[2]])
        ins = [spend_in(sa, ba[2], 55, labels[2]), dummy]
        proofs, pub = prove(labels[2], ins, [(Pa, 3, 55), (Pa, 4, 0)], apath=approved.witness([labels[1]]))
        assert pub[32:64] != approved.root()              # the proof is about another tree: the node's root check refuses it
        assert not ob.verify(vk, pub[:32] + approved.root() + pub[64:], proofs)
        approved.approve([labels[2]])
        proofs, pub = prove(labels[2], ins, [(Pa, 3, 55), (Pa, 4, 0)])
        assert ob.verify(vk, pub, proofs) and pub[32:64] == approved.root()
    finally:
        PK.close()
    # 10. the same approved root serves a labeled association withdrawal of the labeled deposit
    rng2 = random.Random(413)
    tw = [rng2.randrange(1, R) for _ in range(5)]
    lpk, lvk = ob.setup_labeled_association(ctx, 32, *tw)
    LPK = ob.ProvingKey(ctx, lpk)
    try:
        sib, bits = tree.paths([l_label[0]])
        asib, abits = approved.witness(l_label)
        u64 = lambda x: struct.pack("<Q", x)
        proofs, pub = LPK.prove_labeled_association(fr1(token), fr1(1), u64(15), fr([7]), fr([8]), u64(40), l_label, sib, bits,
                                                    fr([9]), fr([10]), asib, abits, cport.frs([3, 4]))
        assert ob.verify(lvk, pub, proofs) and pub[32 * 3:32 * 4] == approved.root()
    finally:
        LPK.close()
