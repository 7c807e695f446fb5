"""The labeled association withdraw statement (oracle/labeled_association_circuit.py == csrc/withdraw_circuit.hpp:
LabeledAssociationBuilder): the spec and its soundness mutations, the library's R1CS export, the GPU witness, setup, ceremony
key and batched prover against the oracle, the provider's approved-label tree (ApprovedLabels) against the spec tree, and a
chain of labeled deposits, partial withdrawals and approvals in one pool tree."""
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
from oracle import labeled_association_circuit as lac
from oracle import labeled_circuit as lc
from oracle import withdraw_circuit as wc
from tests.helpers import pk_blob, vk_blob

R = bn.R
GOLD = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "labeled_association_vectors.json")))
U64 = (1 << 64) - 1
STATEMENTS = ("withdraw", "deposit", "transfer", "association", "exclusion", "labeled", "labeled_association")


# ---- rows: one proof's inputs as ints ---------------------------------------------------------------------------------------
def row(token, recipient, withdrawn, nullifier, secret, amount, label, sibs, bits, cnull, csecret, asibs, abits):
    """bits / abits: path words, bit l set when the level-l node is a right child."""
    return dict(token=token, recipient=recipient, withdrawn=withdrawn, nullifier=nullifier, secret=secret, amount=amount, label=label,
                sibs=sibs, bits=bits, cnull=cnull, csecret=csecret, asibs=asibs, abits=abits)


def bit_list(word, depth):
    return [(word >> l) & 1 for l in range(depth)]


def bit_word(bits):
    return sum(b << l for l, b in enumerate(bits))


def spec_witness(r):
    d = len(r["sibs"])
    return lac.witness(r["nullifier"], r["secret"], r["recipient"], r["token"], r["withdrawn"], r["amount"], r["label"], r["sibs"],
                       bit_list(r["bits"], d), r["cnull"], r["csecret"], r["asibs"], bit_list(r["abits"], d))


def note_row(rng, depth, label, approved, amount=None, withdrawn=None, path_of=None):
    """A random note of `label` at a random pool position (random pool siblings: the root is derived), withdrawing
    `withdrawn` of `amount` (random by default), with the path of approved label `path_of` (default: its own label)."""
    amount = rng.randrange(1 << 64) if amount is None else amount
    withdrawn = rng.randrange(amount + 1) if withdrawn is None else withdrawn
    asibs, abits = approved.path(label if path_of is None else path_of)
    return row(rng.randrange(R), rng.randrange(1 << 160), withdrawn, rng.randrange(R), rng.randrange(R), amount, label,
               [rng.randrange(R) for _ in range(depth)], rng.randrange(1 << depth), rng.randrange(R), rng.randrange(R), asibs,
               bit_word(abits))


def edge_rows(rng, depth):
    """Satisfying rows at the edges: full and zero withdrawals, amount 2^64 - 1, labels 0 and 2^depth - 1, the approved label
    first, in the middle and last of the set."""
    top = (1 << depth) - 1
    mid = min(5, top - 1)
    sets = lac.ApprovedTree(depth, [0, mid, top]), lac.ApprovedTree(depth, [top, 0])
    return [note_row(rng, depth, 0, sets[0], amount=1000, withdrawn=1000),
            note_row(rng, depth, top, sets[0], amount=1000, withdrawn=0),
            note_row(rng, depth, mid, sets[0], amount=U64, withdrawn=U64),
            note_row(rng, depth, top, sets[1], amount=U64, withdrawn=1),
            note_row(rng, depth, 0, sets[1], amount=U64, withdrawn=0),
            note_row(rng, depth, mid, lac.ApprovedTree(depth, [mid]), amount=0, withdrawn=0)]


def valid_rows(rng, batch, depth):
    """Rows whose label is on a random approved list."""
    rows = []
    for _ in range(batch):
        labels = sorted(set(rng.randrange(1 << depth) for _ in range(rng.randrange(1, min(4, 1 << depth) + 1))))
        rows.append(note_row(rng, depth, rng.choice(labels), lac.ApprovedTree(depth, labels)))
    return rows


def random_rows(rng, batch, depth):
    """Rows of uniformly random inputs (amounts and labels anywhere in their integer types): the witness map is defined for
    them too."""
    u64 = lambda: rng.choice([rng.randrange(1 << 64), rng.randrange(1 << 34)])
    return [row(rng.randrange(R), rng.randrange(R), u64(), rng.randrange(R), rng.randrange(R), u64(), rng.randrange(1 << 32),
                [rng.randrange(R) for _ in range(depth)], rng.randrange(1 << 32), rng.randrange(R), rng.randrange(R),
                [rng.randrange(R) for _ in range(depth)], rng.randrange(1 << 32)) for _ in range(batch)]


def pack(rows):
    """The thirteen input buffers of og_labeled_association_witness / og_groth16_prove_labeled_association, in C ABI order."""
    f = cport.frs
    col = lambda k: [r[k] for r in rows]
    return (f(col("token")), f(col("recipient")), col("withdrawn"), f(col("nullifier")), f(col("secret")), col("amount"), col("label"),
            f([x for r in rows for x in r["sibs"]]), col("bits"), f(col("cnull")), f(col("csecret")),
            f([x for r in rows for x in r["asibs"]]), col("abits"))


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
def test_labeled_association_sizes():
    for depth in (1, 2, 32):
        L = lac.Layout(depth)
        assert (L.n_vars, L.n_constraints) == (4975 + 1464 * depth, 4969 + 1462 * depth)
    expect = {32: (51823, 51753, 16), 2: (7903, 7893, 13), 1: (6439, 6431, 13)}
    for depth, (nv, nc, log_m) in expect.items():
        cs = lac.build_r1cs(depth)
        assert (cs.n_vars, cs.n_constraints, cs.n_pub) == (nv, nc, 7), depth
        assert g16.domain_log(cs.n_constraints, cs.n_pub) == log_m, depth
        assert ob.labeled_association_r1cs_info(depth) == dict(n_constraints=nc, n_vars=nv, n_pub=7, log_m=log_m), depth
    for bad in (0, 33):
        with pytest.raises(ob.OwshenB200Error):
            ob.labeled_association_r1cs_info(bad)


def test_seven_statement_shapes_are_distinct():
    """The prover recognises a key by (n_pub, n_vars, n_constraints): no two (statement, depth) pairs of the seven share one."""
    seen = {}
    for stmt in STATEMENTS:
        for d in (range(1, 33) if stmt != "deposit" else (0,)):
            i = api._statement_r1cs_info(stmt, d)
            shape = (i["n_pub"], i["n_vars"], i["n_constraints"])
            assert shape not in seen, (stmt, d, seen.get(shape))
            seen[shape] = (stmt, d)
    assert sum(1 for s in seen if s[0] == 7) == 64            # n_pub = 7: the labeled and labeled association statements


def test_labeled_association_r1cs_export_matches_spec():
    for depth in (1, 2, 32):
        cs = lac.build_r1cs(depth)
        for m in "ABC":
            assert ob.labeled_association_r1cs_export(depth, m) == cs.csr(m), (depth, m)


@pytest.fixture(scope="module")
def cs2():
    return lac.build_r1cs(2)


def test_labeled_association_witnesses_satisfy(cs2):
    rng = random.Random(180)
    for depth, cs in ((2, cs2), (3, lac.build_r1cs(3))):
        for r in edge_rows(rng, depth) + valid_rows(rng, 3, depth):
            w = spec_witness(r)
            assert cs.is_satisfied(w), (r["label"], r["amount"], r["withdrawn"])
            assert w[lac.V_NHASH] == mimc7.multi_hash([r["nullifier"]], key=1)
            assert w[lac.V_ALEAF] == r["label"] + 1
            change = r["amount"] - r["withdrawn"]
            assert w[lac.V_CHANGE_CM] == lc.leaf(lc.precommitment(r["cnull"], r["csecret"]), r["token"], change, r["label"])
            pool = mimc7.merkle_path_nodes(lc.leaf(lc.precommitment(r["nullifier"], r["secret"]), r["token"], r["amount"], r["label"]),
                                           r["sibs"], bit_list(r["bits"], depth))
            assert w[lac.V_ROOT] == pool[-1]
    # the full depth-2 tree (every leaf non-empty), in any order: each label withdraws
    full = lac.ApprovedTree(2, [2, 0, 3, 1])
    for label in range(4):
        w = spec_witness(note_row(rng, 2, label, full))
        assert cs2.is_satisfied(w) and w[lac.V_AROOT] == full.root(), label
    # the spec's note part is the labeled statement's: same public note values as a labeled witness of the same note
    r = note_row(rng, 2, 1, full, amount=1000, withdrawn=250)
    w = spec_witness(r)
    wl = lc.witness(r["nullifier"], r["secret"], r["recipient"], r["token"], r["withdrawn"], r["amount"], r["label"], r["sibs"],
                    bit_list(r["bits"], 2), r["cnull"], r["csecret"], 1, 3, [0, 0], [0, 0])
    assert [w[k] for k in (1, 2, 3, 5, 6, 7)] == [wl[k] for k in (1, 2, 3, 5, 6, 7)]


def test_labeled_association_mutations_are_unsatisfied(cs2):
    rng = random.Random(182)
    L = lac.Layout(2)
    approved = lac.ApprovedTree(2, [1, 3])                   # leaves 2, 4, 0, 0
    good = note_row(rng, 2, 3, approved, amount=1000, withdrawn=300)
    w0 = spec_witness(good)
    assert failing(cs2, w0) == [] and w0[lac.V_AROOT] == approved.root()
    # an unapproved label with an approved label's path, against the provider's root
    for path_of in (1, 3):
        w = spec_witness(note_row(rng, 2, 2, approved, path_of=path_of))
        assert w[lac.V_AROOT] != approved.root()
        w[lac.V_AROOT] = approved.root()
        assert failing(cs2, w) == [L.row_assoc_root], path_of
    # label = r - 1 makes assoc_leaf 0, which an empty slot holds: only the label's range check stops it
    asibs, abits = approved.tree.path(2)
    w = spec_witness(dict(good, label=R - 1, asibs=asibs, abits=bit_word(abits)))
    assert w[lac.V_ALEAF] == 0 and w[lac.V_AROOT] == approved.root()
    assert failing(cs2, w) == [L.packed_row(lac.LABEL)]
    # an assoc_leaf other than label + 1: the leaf of approved label 3 carried by a note of label 2
    w = spec_witness(note_row(rng, 2, 2, approved, path_of=3))
    w[lac.V_ALEAF] = 4
    sibs, bits = approved.path(3)
    w[lac.V_AROOT] = lac.levels_witness(w, L, lac.ASSOC, 4, sibs, bits)
    assert w[lac.V_AROOT] == approved.root()
    assert failing(cs2, w) == [L.row_assoc_leaf]
    # an overdraw: withdrawn > amount leaves change = r - 1
    assert failing(cs2, spec_witness(dict(good, withdrawn=1001))) == [L.packed_row(lac.CHANGE)]
    # withdrawn = r - k would make change = amount + k (a mint of k): only the withdrawn range check stops it
    for k in (1, 7):
        assert failing(cs2, spec_witness(dict(good, withdrawn=R - k))) == [L.packed_row(lac.WITHDRAWN)], k
    # amount >= 2^64
    assert failing(cs2, spec_witness(dict(good, amount=(1 << 64) + 5, withdrawn=10))) == [L.packed_row(lac.AMOUNT)]
    # change_commitment under another label (or token, or amount) than the statement's
    cpre = lc.precommitment(good["cnull"], good["csecret"])
    assert w0[lac.V_CHANGE_CM] == lc.leaf(cpre, good["token"], 700, 3)
    for token, change, label in ((good["token"], 700, 1), (good["token"], 700, 2), (good["token"] + 1, 700, 3), (good["token"], 701, 3)):
        w = list(w0)
        w[lac.V_CHANGE_CM] = lc.leaf(cpre, token, change, label)
        assert failing(cs2, w) == [L.row_change_cm], (token, change, label)
    # a wrong nullifier hash: the row that binds the hash's output
    w = list(w0)
    w[lac.V_NHASH] = (w[lac.V_NHASH] + 1) % R
    assert failing(cs2, w) == [1 + L.perm]
    # recipient_sq
    w = list(w0)
    w[lac.V_RSQ] = (w[lac.V_RSQ] + 1) % R
    assert failing(cs2, w) == [0]


def golden_row(g):
    return row(int(g["token"]), int(g["recipient"]), g["withdrawn"], int(g["nullifier"]), int(g["secret"]), g["amount"], g["label"],
               [int(x) for x in g["siblings"]], g["path_bits"], int(g["change_nullifier"]), int(g["change_secret"]),
               [int(x) for x in g["assoc_siblings"]], g["assoc_path_bits"])


def test_labeled_association_golden_proof_reproduced_by_c_port():
    g = GOLD
    cs = lac.build_r1cs(g["depth"])
    pkb, vkb = cport.setup_bytes(cs, *[int(x) for x in g["toxic"]])
    assert hashlib.sha256(pkb["a"] + pkb["b1"] + pkb["b2"] + pkb["l"] + pkb["h"]).hexdigest() == g["pk_queries_sha256"]
    v = g["vk"]
    assert (vkb["alpha1"] + vkb["beta2"] + vkb["gamma2"] + vkb["delta2"] + vkb["ic"]).hex() == v["alpha1"] + v["beta2"] + v["gamma2"] + v["delta2"] + v["ic"]
    w = spec_witness(golden_row(g))
    assert cs.is_satisfied(w)
    assert w[lac.V_AROOT] == lac.ApprovedTree(g["depth"], g["approved"]).root()
    wit = cport.frs(w)
    assert hashlib.sha256(wit).hexdigest() == g["witness_sha256"]
    assert cport.unfr(wit[32:32 * 8]) == [int(x) for x in g["public"]]
    assert cport.Prover(cs, pkb).prove(wit, int(g["r"]), int(g["s"])).hex() == g["proof"]
    assert ob.verify(vk_blob(vkb, 7), wit[32:32 * 8], bytes.fromhex(g["proof"]))


def test_labeled_association_inputs_are_validated_at_the_boundary():
    """Labels outside uint32, amounts outside uint64 and arrays of the wrong length are refused before any call into the
    library."""
    rows = valid_rows(random.Random(183), 2, 2)
    args = lambda p: api._statement_args("labeled_association", "labeled_association_witness", 2, 2, p)
    assert len(args(pack(rows))) == 13
    p = pack(rows)
    for k, bad in ((2, [1 << 64, 0]), (5, [0, -1]), (6, [1 << 32, 0]), (6, [-1, 0]), (6, p[6][:1]), (7, p[7][:-32]), (8, p[8] + [0]),
                   (11, p[11] + bytes(32)), (12, p[12][:1])):
        q = list(p)
        q[k] = bad
        with pytest.raises(ValueError):
            args(q)


# ---- GPU -----------------------------------------------------------------------------------------------------------------
_KEYS = {}


def keys(ctx, depth):
    """(pk, vk, r1cs, oracle pk bytes, oracle vk bytes) of the depth-`depth` labeled association statement, made once."""
    if depth not in _KEYS:
        rng = random.Random(190 + depth)
        tw = [rng.randrange(1, R) for _ in range(5)]
        pk, vk = ob.setup_labeled_association(ctx, depth, *tw)
        cs = lac.build_r1cs(depth)
        pkb, vkb = cport.setup_bytes(cs, *tw)
        _KEYS[depth] = (pk, vk, cs, pkb, vkb)
    return _KEYS[depth]


def proofs_verify(vk, proofs, pub, batch):
    return [ob.verify(vk, pub[224 * i:224 * i + 224], proofs[256 * i:256 * i + 256]) for i in range(batch)]


@pytest.mark.gpu
def test_labeled_association_witness_matches_oracle(ctx):
    rng = random.Random(192)
    # depth 2: 40 rows with every edge row, the soundness mutations' rows and random inputs anywhere in their types
    approved = lac.ApprovedTree(2, [1, 3])
    good = note_row(rng, 2, 3, approved, amount=1000, withdrawn=300)
    mutated = [note_row(rng, 2, 2, approved, path_of=1), note_row(rng, 2, 0, approved, path_of=3), dict(good, withdrawn=1001),
               dict(good, amount=0, withdrawn=U64), dict(good, amount=U64, withdrawn=0), dict(good, amount=5, withdrawn=U64),
               dict(good, label=(1 << 32) - 1), dict(good, label=(1 << 32) - 2)]
    rows = edge_rows(rng, 2) + mutated + valid_rows(rng, 6, 2)
    rows += random_rows(rng, 40 - len(rows), 2)
    assert len(rows) == 40
    assert ctx.labeled_association_witness(2, *pack(rows)) == oracle_witnesses(rows)
    rows = edge_rows(rng, 32)[:4] + random_rows(rng, 2, 32)
    assert ctx.labeled_association_witness(32, *pack(rows)) == oracle_witnesses(rows)
    # a field input >= r in any of the eight field arrays
    rows = valid_rows(rng, 2, 2)
    for k in (0, 1, 3, 4, 7, 9, 10, 11):
        p = list(pack(rows))
        p[k] = R.to_bytes(32, "little") + p[k][32:]
        with pytest.raises(ob.OwshenB200Error) as e:
            ctx.labeled_association_witness(2, *p)
        assert e.value.code == -4 or "encoding" in str(e.value).lower(), k


@pytest.mark.gpu
def test_setup_labeled_association_matches_oracle(ctx):
    for depth in (2, 32):
        pk, vk, cs, pkb, vkb = keys(ctx, depth)
        assert pk == pk_blob(cs, pkb, 0), depth
        assert vk == vk_blob(vkb, 7), depth


@pytest.mark.gpu
def test_labeled_association_key_from_ceremony(ctx):
    """One phase-1 contribution (t, a, b), the depth-2 key, then a phase-2 contribution d: the development setup with the
    product secrets (t, a, b, 1, d) (DESIGN.md section 4b)."""
    rng = random.Random(193)
    t, a, b, d = (rng.randrange(1, R) for _ in range(4))
    acc0 = ob.ptau_new(ctx, 13)                           # the depth-2 labeled association domain is 2^13
    acc1, rec = ob.ptau_contribute(ctx, acc0, [t, a, b], [rng.randrange(1, R) for _ in range(3)])
    assert ob.ptau_verify(ctx, acc0, acc1, rec)
    pk0, vk0 = ob.ptau_prepare_labeled_association(ctx, acc1, 2)
    assert (pk0, vk0) == ob.setup_labeled_association(ctx, 2, t, a, b, 1, 1)
    pk, vk, rec2 = ob.phase2_contribute(ctx, pk0, vk0, d, rng.randrange(1, R))
    assert ob.phase2_verify(ctx, pk0, vk0, pk, vk, rec2)
    assert (pk, vk) == ob.setup_labeled_association(ctx, 2, t, a, b, 1, d)
    cs = lac.build_r1cs(2)
    pkb, vkb = cport.setup_bytes(cs, t, a, b, 1, d)
    assert pk == pk_blob(cs, pkb, 0) and vk == vk_blob(vkb, 7)
    PK = ob.ProvingKey(ctx, pk)
    try:
        assert (PK.labeled_association_depth, PK.labeled_depth, PK.association_depth) == (2, None, None)
    finally:
        PK.close()


@pytest.mark.gpu
@pytest.mark.parametrize("depth,batch", [(2, 40), (32, 3)])
def test_prove_labeled_association_matches_oracle(ctx, monkeypatch, depth, batch):
    """Default settings, then chunks below the batch on two lanes: both byte for byte the oracle C prover's."""
    pk, vk, cs, pkb, vkb = keys(ctx, depth)
    rng = random.Random(194 + depth)
    rows = (edge_rows(rng, depth) + valid_rows(rng, batch, depth))[:batch]
    rs = cport.frs([rng.randrange(R) for _ in range(2 * batch)])
    wit = oracle_witnesses(rows)
    exp = cport.Prover(cs, pkb).prove_batch(wit, rs)
    results = []
    for env in (dict(), dict(OG_CHUNK=3 if depth == 2 else 2, OG_LANES=2)):
        set_env(monkeypatch, **env)
        PK = ob.ProvingKey(ctx, pk)
        try:
            assert (PK.n_vars, PK.n_pub, PK.depth, PK.labeled_association_depth, PK.labeled_depth) == (cs.n_vars, 7, 0, depth, None)
            results.append(PK.prove_labeled_association(*pack(rows), rs))
        finally:
            PK.close()
    set_env(monkeypatch)
    nv = cs.n_vars
    for proofs, pub in results:
        assert proofs == exp
        assert pub == b"".join(wit[32 * nv * i + 32:32 * nv * i + 32 * 8] for i in range(batch))
    proofs, pub = results[0]
    assert all(proofs_verify(vk, proofs, pub, batch))
    for k in (3, 5, 6):                                   # another association root, withdrawn or change commitment
        bad = bytearray(pub[:224]); bad[32 * k] ^= 1
        assert not ob.verify(vk, bytes(bad), proofs[:256]), k


@pytest.mark.gpu
def test_prove_labeled_association_dev_matches_host_entry_point(ctx):
    import torch
    pk = keys(ctx, 2)[0]
    rng = random.Random(195)
    batch = 5
    rows = valid_rows(rng, batch, 2)
    rs = cport.frs([rng.randrange(R) for _ in range(2 * batch)])
    p = pack(rows)
    PK = ob.ProvingKey(ctx, pk)
    try:
        proofs, pub = PK.prove_labeled_association(*p, rs)
        fmt = {2: "Q", 5: "Q", 6: "I", 8: "I", 12: "I"}
        raw = [struct.pack(f"<{len(x)}{fmt[k]}", *x) if k in fmt else x for k, x in enumerate(p)]
        dev = lambda b: torch.frombuffer(bytearray(b), dtype=torch.uint8).to("cuda")
        d_in = [dev(x) for x in raw + [rs]]
        d_pr = torch.zeros(256 * batch, dtype=torch.uint8, device="cuda")
        d_pub = torch.zeros(224 * batch, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        rc = api.lib().og_groth16_prove_labeled_association_dev(ctx._h, PK._h, *[api._ptr(t) for t in d_in[:13]], batch,
                                                                api._ptr(d_in[13]), api._ptr(d_pr), api._ptr(d_pub))
        assert rc == 0
        ctx.sync()
        assert bytes(d_pr.cpu().numpy()) == proofs and bytes(d_pub.cpu().numpy()) == pub
    finally:
        PK.close()


@pytest.mark.gpu
def test_labeled_association_golden_proof(ctx):
    g = GOLD
    pk, vk = ob.setup_labeled_association(ctx, g["depth"], *[int(x) for x in g["toxic"]])
    v = g["vk"]
    assert vk[12:].hex() == v["alpha1"] + v["beta2"] + v["gamma2"] + v["delta2"] + v["ic"]
    rs = bn.fr_to_bytes(int(g["r"])) + bn.fr_to_bytes(int(g["s"]))
    PK = ob.ProvingKey(ctx, pk)
    try:
        proofs, pub = PK.prove_labeled_association(*pack([golden_row(g)]), rs)
    finally:
        PK.close()
    assert proofs.hex() == g["proof"]
    assert cport.unfr(pub) == [int(x) for x in g["public"]]
    assert ob.verify(vk, pub, proofs)


# every statement's prover: (name, number of input arrays)
_PROVERS = (("withdraw", 5), ("deposit", 3), ("transfer", 11), ("association", 7), ("exclusion", 9), ("labeled", 15),
            ("labeled_association", 13))


@pytest.mark.gpu
def test_seven_provers_refuse_each_others_keys(ctx):
    import torch
    d_buf = torch.zeros(1 << 16, dtype=torch.uint8, device="cuda")
    d = api._ptr(d_buf)                                   # every device argument of the _dev entry points
    h = bytes(1 << 16)                                    # every host input of the host entry points
    rng = random.Random(196)
    tw = [rng.randrange(1, R) for _ in range(5)]
    all_keys = {"withdraw": ob.setup_withdraw(ctx, 2, *tw)[0], "deposit": ob.setup_deposit(ctx, *tw)[0],
                "transfer": ob.setup_transfer(ctx, 2, *tw)[0], "association": ob.setup_association(ctx, 2, *tw)[0],
                "exclusion": ob.setup_exclusion(ctx, 2, *tw)[0], "labeled": ob.setup_labeled(ctx, 2, *tw)[0],
                "labeled_association": keys(ctx, 2)[0]}
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
            if owner != "labeled_association":
                with pytest.raises(ob.OwshenB200Error):
                    PK.prove_labeled_association(*pack(valid_rows(rng, 1, 2)), bytes(64))
        finally:
            PK.close()
    PK = ob.ProvingKey(ctx, all_keys["labeled_association"])
    try:
        rows = valid_rows(rng, 2, 2)
        assert len(PK.prove_labeled_association(*pack(rows), cport.frs([rng.randrange(R) for _ in range(4)]))[0]) == 512
    finally:
        PK.close()


@pytest.mark.gpu
def test_approved_labels_match_spec_tree(ctx):
    """Construction (unsorted, with duplicates), approve() appends (new labels, duplicates of approved ones, duplicates within
    the batch), witness paths and every refusal, against the spec tree of leaves label + 1."""
    from owshen_b200.kvstore import RamKvStore
    as_int = lambda b: int.from_bytes(b, "little")
    for depth in (2, 32):
        top = (1 << depth) - 1
        first = [3, top, 0, 3] if depth == 32 else [3, 0, 3]
        al = ob.ApprovedLabels(ctx, depth, first)
        spec = lac.ApprovedTree(depth, sorted(set(first)))
        assert as_int(al.root()) == spec.root() and len(al) == len(spec.labels) and al.labels == spec.labels, depth
        assert 3 in al and 0 in al and 1 not in al
        more = [1, 0, 1 << 20, 1] if depth == 32 else [1, 0, 1]
        assert al.approve(more) == sorted(set(more) - set(first))
        spec.approve(sorted(set(more) - set(first)))
        assert as_int(al.root()) == spec.root() and al.labels == spec.labels, depth
        assert al.approve([0, 3]) == [] and as_int(al.root()) == spec.root()
        sibs, bits = al.witness([1, 3, 1])
        for k, label in enumerate([1, 3, 1]):
            s, b = spec.path(label)
            assert cport.unfr(sibs[32 * depth * k:32 * depth * (k + 1)]) == s and bits[k] == bit_word(b), (depth, label)
        missing = 2 if depth == 2 else 7
        with pytest.raises(ValueError, match=rf"\[{missing}, {top + 1}\]"):
            al.witness([missing, 1, top + 1, missing])
        root = al.root()
        for bad in ([top + 1], [-1], [0, 1 << 32]):
            with pytest.raises(ValueError):
                al.approve(bad)
            with pytest.raises(ValueError):
                ob.ApprovedLabels(ctx, depth, bad)
        assert al.root() == root and al.labels == spec.labels            # a refused batch changes nothing
    # the full depth-2 set, and an empty one
    assert as_int(ob.ApprovedLabels(ctx, 2, [3, 2, 1, 0]).root()) == lac.ApprovedTree(2, [0, 1, 2, 3]).root()
    empty = ob.ApprovedLabels(ctx, 2, [])
    assert len(empty) == 0 and as_int(empty.root()) == mimc7.MerkleTree(2).root()
    store = RamKvStore()
    ob.ApprovedLabels(ctx, 2, [1], store=store)
    with pytest.raises(ValueError):
        ob.ApprovedLabels(ctx, 2, [2], store=store)
    for depth in (0, 33):
        with pytest.raises(ValueError):
            ob.ApprovedLabels(ctx, depth, [])


@pytest.mark.gpu
def test_labeled_deposits_withdrawals_and_approvals_chain(ctx):
    """Labeled deposits interleaved with plain ones in one depth-32 pool tree; a provider approves two of three.  An approved
    deposit withdraws in part and its change note is appended; the change note withdraws again under the same label.  The
    unapproved deposit gets no witness, and a forced neighbouring path gives a proof that fails against the provider's root;
    once approved it withdraws, with the nullifier hash the labeled statement gives the same note."""
    rng = random.Random(197)
    depth = 32
    as_int = lambda b: int.from_bytes(b, "little")
    token = rng.randrange(R)
    pool, spec = ob.MerkleTree(ctx, depth), mimc7.MerkleTree(depth)

    def plain(n):
        cms = [mimc7.multi_hash([rng.randrange(R), rng.randrange(R)]) for _ in range(n)]
        pool.insert_batch(cms)
        for c in cms:
            spec.insert(c)

    def labeled(notes):
        pres = ctx.labeled_precommitments(cport.frs([n[0] for n in notes]), cport.frs([n[1] for n in notes]))
        labels = ob.deposit_labeled(pool, pres, cport.frs([token] * len(notes)), [n[2] for n in notes])
        for n, label in zip(notes, labels):
            spec.insert(lc.leaf(lc.precommitment(n[0], n[1]), token, n[2], label))
        return labels

    plain(2)
    notes = [(rng.randrange(R), rng.randrange(R), rng.randrange(1 << 40, 1 << 64)) for _ in range(3)]
    labels = labeled(notes[:2])
    plain(1)
    labels += labeled(notes[2:])
    assert labels == [2, 3, 5] and pool.n_leaves == 6
    assert as_int(pool.root()) == spec.root()
    a, b, c = labels
    provider = ob.ApprovedLabels(ctx, depth, [b, a, 1 << 20])
    pk, vk = keys(ctx, depth)[:2]
    PK = ob.ProvingKey(ctx, pk)

    def withdraw(note, index, label, withdrawn, asibs=None, abits=None):
        """One labeled association withdrawal of the note at pool leaf `index` -> (change note, public inputs, verifies
        against the provider's current root)."""
        if asibs is None:
            asibs, abits = provider.witness([label])
        sibs, bits = pool.paths([index])
        change = (rng.randrange(R), rng.randrange(R), note[2] - withdrawn)
        recipient = rng.randrange(1 << 160)
        proofs, pub = PK.prove_labeled_association(cport.frs([token]), cport.frs([recipient]), [withdrawn], cport.frs([note[0]]),
                                                   cport.frs([note[1]]), [note[2]], [label], sibs, bits, cport.frs([change[0]]),
                                                   cport.frs([change[1]]), asibs, abits, cport.frs([rng.randrange(R), rng.randrange(R)]))
        p = cport.unfr(pub)
        assert p[:3] == [as_int(pool.root()), mimc7.multi_hash([note[0]], key=1), recipient] and p[4:6] == [token, withdrawn]
        assert p[6] == lc.leaf(lc.precommitment(change[0], change[1]), token, change[2], label)
        published = pub[:96] + provider.root() + pub[128:]
        return change, pub, ob.verify(vk, published, proofs)

    try:
        # a partial withdrawal of deposit B; the node appends its change commitment
        change1, pub, ok = withdraw(notes[1], b, b, notes[1][2] // 3)
        assert ok and pub[96:128] == provider.root()
        i1 = pool.insert(pub[32 * 6:32 * 7])
        plain(1)
        # the change note withdraws again at its own index under B's label
        change2, pub, ok = withdraw(change1, i1, b, 12345)
        assert ok
        pool.insert(pub[32 * 6:32 * 7])
        # deposit C is not approved: no witness, and the path of an approved neighbour derives another association root
        with pytest.raises(ValueError, match=str(c)):
            provider.witness([c])
        for neighbour in (b, 1 << 20):
            asibs, abits = provider.witness([neighbour])
            _, pub, ok = withdraw(notes[2], c, c, 1, asibs, abits)
            assert pub[96:128] != provider.root() and not ok, neighbour
        # the provider clears C; it withdraws, with the nullifier hash the labeled statement gives the same note
        assert provider.approve([c, a]) == [c]
        _, pub, ok = withdraw(notes[2], c, c, 1)
        assert ok
        lpk = ob.setup_labeled(ctx, depth, *[rng.randrange(1, R) for _ in range(5)])[0]
        LPK = ob.ProvingKey(ctx, lpk)
        try:
            blocklist = ob.ExclusionSet(ctx, depth, [a])
            low, nxt, xsibs, xbits = blocklist.witness([c])
            sibs, bits = pool.paths([c])
            lpub = LPK.prove_labeled(cport.frs([token]), cport.frs([1]), [1], cport.frs([notes[2][0]]), cport.frs([notes[2][1]]),
                                     [notes[2][2]], [c], sibs, bits, cport.frs([5]), cport.frs([6]), low, nxt, xsibs, xbits,
                                     cport.frs([rng.randrange(R), rng.randrange(R)]))[1]
        finally:
            LPK.close()
        assert lpub[32:64] == pub[32:64] == bn.fr_to_bytes(mimc7.multi_hash([notes[2][0]], key=1))
    finally:
        PK.close()
