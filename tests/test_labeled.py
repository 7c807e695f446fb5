"""Labeled value notes and the labeled withdraw statement (oracle/labeled_circuit.py == csrc/withdraw_circuit.hpp:
LabeledBuilder): the note format and its domain separation, the spec and its soundness mutations, the library's R1CS export,
the two GPU note hashes, GPU witness, setup, ceremony key and batched prover against the oracle, and a chain of labeled
deposits, partial withdrawals and blocklist versions in one pool tree."""
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
from oracle import exclusion_circuit as xc
from oracle import groth16 as g16
from oracle import labeled_circuit as lc
from oracle import transfer_circuit as tc
from oracle import withdraw_circuit as wc
from tests.helpers import pk_blob, vk_blob

R = bn.R
GOLD = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "labeled_vectors.json")))
U64 = (1 << 64) - 1
STATEMENTS = ("withdraw", "deposit", "transfer", "association", "exclusion", "labeled")


# ---- rows: one proof's inputs as ints ---------------------------------------------------------------------------------------
def row(token, recipient, withdrawn, nullifier, secret, amount, label, sibs, bits, cnull, csecret, low, next_, xsibs, xbits):
    """bits / xbits: path words, bit l set when the level-l node is a right child."""
    return dict(token=token, recipient=recipient, withdrawn=withdrawn, nullifier=nullifier, secret=secret, amount=amount, label=label,
                sibs=sibs, bits=bits, cnull=cnull, csecret=csecret, low=low, next=next_, xsibs=xsibs, xbits=xbits)


def bit_list(word, depth):
    return [(word >> l) & 1 for l in range(depth)]


def bit_word(bits):
    return sum(b << l for l, b in enumerate(bits))


def spec_witness(r):
    d = len(r["sibs"])
    return lc.witness(r["nullifier"], r["secret"], r["recipient"], r["token"], r["withdrawn"], r["amount"], r["label"], r["sibs"],
                      bit_list(r["bits"], d), r["cnull"], r["csecret"], r["low"], r["next"], r["xsibs"], bit_list(r["xbits"], d))


def note_row(rng, depth, label, blocklist, amount=None, withdrawn=None, leaf=None):
    """A random note of `label` at a random pool position (random pool siblings: the root is derived), withdrawing
    `withdrawn` of `amount` (random by default), with the blocklist path of `leaf` (default: the leaf that brackets it)."""
    amount = rng.randrange(1 << 64) if amount is None else amount
    withdrawn = rng.randrange(amount + 1) if withdrawn is None else withdrawn
    j = blocklist.bracket(label) if leaf is None else leaf
    xsibs, xbits = blocklist.tree.path(j)
    return row(rng.randrange(R), rng.randrange(1 << 160), withdrawn, rng.randrange(R), rng.randrange(R), amount, label,
               [rng.randrange(R) for _ in range(depth)], rng.randrange(1 << depth), rng.randrange(R), rng.randrange(R),
               blocklist.keys[j], blocklist.keys[j + 1], xsibs, bit_word(xbits))


def edge_rows(rng, depth):
    """Satisfying rows at the edges: full and zero withdrawals, amount 2^64 - 1, labels 0 and 2^depth - 1, an empty
    blocklist, a label whose neighbours are both flagged."""
    top = (1 << depth) - 1
    mid = min(5, top - 1)
    empty = xc.BlocklistTree(depth, [])
    return [note_row(rng, depth, 0, empty, amount=1000, withdrawn=1000),
            note_row(rng, depth, top, empty, amount=1000, withdrawn=0),
            note_row(rng, depth, mid, xc.BlocklistTree(depth, [mid - 1, mid + 1]), amount=U64, withdrawn=U64),
            note_row(rng, depth, 0, xc.BlocklistTree(depth, [top]), amount=U64, withdrawn=1),
            note_row(rng, depth, top, xc.BlocklistTree(depth, [0]), amount=U64, withdrawn=0),
            note_row(rng, depth, 1, xc.BlocklistTree(depth, [0, top]), amount=0, withdrawn=0)]


def valid_rows(rng, batch, depth):
    """Rows whose label is unflagged in a random blocklist."""
    rows = []
    for _ in range(batch):
        flagged = sorted(set(rng.randrange(1 << depth) for _ in range(rng.randrange(0, min(4, (1 << depth) - 1) + 1))))
        free = [i for i in ([rng.randrange(1 << depth) for _ in range(8)] + list(range(4))) if i not in flagged and i < 1 << depth]
        rows.append(note_row(rng, depth, free[0], xc.BlocklistTree(depth, flagged)))
    return rows


def random_rows(rng, batch, depth):
    """Rows of uniformly random inputs (amounts, labels and keys anywhere in their integer types): the witness map is
    defined for them too."""
    u64 = lambda: rng.choice([rng.randrange(1 << 64), rng.randrange(1 << 34)])
    return [row(rng.randrange(R), rng.randrange(R), u64(), rng.randrange(R), rng.randrange(R), u64(), rng.randrange(1 << 32),
                [rng.randrange(R) for _ in range(depth)], rng.randrange(1 << 32), rng.randrange(R), rng.randrange(R), u64(), u64(),
                [rng.randrange(R) for _ in range(depth)], rng.randrange(1 << 32)) for _ in range(batch)]


def pack(rows):
    """The fifteen input buffers of og_labeled_witness / og_groth16_prove_labeled, in C ABI order."""
    f = cport.frs
    col = lambda k: [r[k] for r in rows]
    return (f(col("token")), f(col("recipient")), col("withdrawn"), f(col("nullifier")), f(col("secret")), col("amount"), col("label"),
            f([x for r in rows for x in r["sibs"]]), col("bits"), f(col("cnull")), f(col("csecret")), col("low"), col("next"),
            f([x for r in rows for x in r["xsibs"]]), col("xbits"))


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
def test_labeled_sizes():
    for depth in (1, 2, 32):
        L = lc.Layout(depth)
        assert (L.n_vars, L.n_constraints) == (5837 + 1464 * depth, 5833 + 1462 * depth)
    expect = {32: (52685, 52617, 16), 2: (8765, 8757, 14), 1: (7301, 7295, 13)}
    for depth, (nv, nc, log_m) in expect.items():
        cs = lc.build_r1cs(depth)
        assert (cs.n_vars, cs.n_constraints, cs.n_pub) == (nv, nc, 7), depth
        assert g16.domain_log(cs.n_constraints, cs.n_pub) == log_m, depth
        assert ob.labeled_r1cs_info(depth) == dict(n_constraints=nc, n_vars=nv, n_pub=7, log_m=log_m), depth
    for bad in (0, 33):
        with pytest.raises(ob.OwshenB200Error):
            ob.labeled_r1cs_info(bad)


def test_six_statement_shapes_are_distinct():
    """The prover recognises a key by (n_pub, n_vars, n_constraints): no two (statement, depth) pairs of the six share one."""
    seen = {}
    for stmt in STATEMENTS:
        for d in (range(1, 33) if stmt != "deposit" else (0,)):
            i = api._statement_r1cs_info(stmt, d)
            shape = (i["n_pub"], i["n_vars"], i["n_constraints"])
            assert shape not in seen, (stmt, d, seen.get(shape))
            seen[shape] = (stmt, d)
    assert sum(1 for s in seen if s[0] == 7) == 32            # n_pub = 7 is the labeled statement's alone


def test_labeled_r1cs_export_matches_spec():
    for depth in (1, 2, 32):
        cs = lc.build_r1cs(depth)
        for m in "ABC":
            assert ob.labeled_r1cs_export(depth, m) == cs.csr(m), (depth, m)


def test_labeled_note_format_and_domain_separation():
    """Key 2: the labeled leaf of (pre, token, amount, label) is not the transfer commitment of the same tuple read as
    (nullifier = pre, secret = token, token = amount, amount = label).  Under key 0 it would be, and a transfer statement
    could spend the deposit from public values alone."""
    rng = random.Random(80)
    nu, se, token, amount, label = rng.randrange(R), rng.randrange(R), rng.randrange(R), rng.randrange(1 << 64), 1
    pre = lc.precommitment(nu, se)
    assert pre == mimc7.multi_hash([nu, se], 2) != mimc7.multi_hash([nu, se], 0)
    leaf = lc.leaf(pre, token, amount, label)
    assert leaf == mimc7.multi_hash([pre, token, amount, label], 2)
    key0 = mimc7.multi_hash([pre, token, amount, label], 0)
    assert leaf != key0
    # the theft: a transfer spending (pre, token, label) of token `amount`, all public at deposit
    cs = tc.build_r1cs(2)
    for pool_leaf, stealable in ((key0, True), (leaf, False)):
        pool = mimc7.MerkleTree(2)
        pool.insert(rng.randrange(R))
        i = pool.insert(pool_leaf)
        sibs, bits = pool.path(i)
        ins = [(pre, token, label, sibs, bit_word(bits)), (rng.randrange(R), rng.randrange(R), 0, [0, 0], 0)]
        outs = [(rng.randrange(R), rng.randrange(R), label), (rng.randrange(R), rng.randrange(R), 0)]
        w = tc.witness(pool.root(), amount, rng.randrange(1 << 160), ins, outs)
        assert w[tc.V_OUT_CM[0]] and cs.is_satisfied(w) == stealable, stealable


@pytest.fixture(scope="module")
def cs2():
    return lc.build_r1cs(2)


def test_labeled_witnesses_satisfy(cs2):
    rng = random.Random(81)
    for depth, cs in ((2, cs2), (3, lc.build_r1cs(3))):
        for r in edge_rows(rng, depth) + valid_rows(rng, 3, depth):
            w = spec_witness(r)
            assert cs.is_satisfied(w), (r["label"], r["amount"], r["withdrawn"])
            assert w[lc.V_NHASH] == mimc7.multi_hash([r["nullifier"]], key=1)
            change = r["amount"] - r["withdrawn"]
            assert w[lc.V_CHANGE_CM] == lc.leaf(lc.precommitment(r["cnull"], r["csecret"]), r["token"], change, r["label"])
            pool = mimc7.merkle_path_nodes(lc.leaf(lc.precommitment(r["nullifier"], r["secret"]), r["token"], r["amount"], r["label"]),
                                           r["sibs"], bit_list(r["bits"], depth))
            assert w[lc.V_ROOT] == pool[-1]
    # the full depth-2 tree: 2^2 - 1 flagged deposits leave one label that can withdraw
    full = xc.BlocklistTree(2, [0, 1, 3])
    w = spec_witness(note_row(rng, 2, 2, full))
    assert cs2.is_satisfied(w) and w[lc.V_XROOT] == full.root()


def test_labeled_mutations_are_unsatisfied(cs2):
    rng = random.Random(82)
    L = lc.Layout(2)
    bl = xc.BlocklistTree(2, [1, 2])                          # keys 0, 2, 3, 2^32 + 1
    good = note_row(rng, 2, 3, bl, amount=1000, withdrawn=300)
    assert failing(cs2, spec_witness(good)) == []
    # a flagged label with either neighbouring leaf: leaf 0 = (0, 2) fails gap_hi, leaf 1 = (2, 3) gap_lo
    assert failing(cs2, spec_witness(note_row(rng, 2, 1, bl, leaf=0))) == [L.packed_row(lc.GAP_HI)]
    assert failing(cs2, spec_witness(note_row(rng, 2, 1, bl, leaf=1))) == [L.packed_row(lc.GAP_LO)]
    # a published leaf that does not bracket x = label + 1
    assert failing(cs2, spec_witness(note_row(rng, 2, 3, bl, leaf=0))) == [L.packed_row(lc.GAP_HI)]
    assert failing(cs2, spec_witness(note_row(rng, 2, 0, bl, leaf=2))) == [L.packed_row(lc.GAP_LO)]
    # an overdraw: withdrawn > amount leaves change = r - 1
    assert failing(cs2, spec_witness(dict(good, withdrawn=1001))) == [L.packed_row(lc.CHANGE)]
    assert failing(cs2, spec_witness(dict(good, amount=0, withdrawn=U64))) == [L.packed_row(lc.CHANGE)]
    # withdrawn = r - 1 would make change = amount + 1 (a mint of 1): only the withdrawn range check stops it
    assert failing(cs2, spec_witness(dict(good, withdrawn=R - 1))) == [L.packed_row(lc.WITHDRAWN)]
    # change_commitment of another label, token or amount than the statement's
    w0 = spec_witness(good)
    cpre = lc.precommitment(good["cnull"], good["csecret"])
    for token, change, label in ((good["token"], 700, 2), (good["token"] + 1, 700, 3), (good["token"], 701, 3), (good["token"], 1000, 3)):
        w = list(w0)
        w[lc.V_CHANGE_CM] = lc.leaf(cpre, token, change, label)
        assert failing(cs2, w) == [L.row_change_cm], (token, change, label)
    assert w0[lc.V_CHANGE_CM] == lc.leaf(cpre, good["token"], 700, 3)
    # label >= 2^32 (a leaf the node never made): its 32 bits do not pack back to the label
    for big in (1 << 32, (1 << 32) + 3, R - 1):
        assert L.packed_row(lc.LABEL) in failing(cs2, spec_witness(dict(good, label=big))), big
    # amount >= 2^64
    assert failing(cs2, spec_witness(dict(good, amount=(1 << 64) + 5, withdrawn=10))) == [L.packed_row(lc.AMOUNT)]
    # recipient_sq
    w = list(w0)
    w[lc.V_RSQ] = (w[lc.V_RSQ] + 1) % R
    assert failing(cs2, w) == [0]
    # the key-0 leaf of the same tuple in the pool: the note does not open under that root
    pre = lc.precommitment(good["nullifier"], good["secret"])
    for key, ok in ((0, False), (2, True)):
        pool = mimc7.MerkleTree(2)
        pool.insert(rng.randrange(R))
        i = pool.insert(mimc7.multi_hash([pre, good["token"], good["amount"], good["label"]], key))
        sibs, bits = pool.path(i)
        w = spec_witness(dict(good, sibs=sibs, bits=bit_word(bits)))
        w[lc.V_ROOT] = pool.root()
        assert failing(cs2, w) == ([] if ok else [L.row_pool_root]), key
    # an exclusion path bit flipped, with the published root claimed
    w = list(w0)
    w[L.level(lc.EXCL, 1)["bit"]] ^= 1
    assert failing(cs2, w)


def golden_row(g):
    return row(int(g["token"]), int(g["recipient"]), g["withdrawn"], int(g["nullifier"]), int(g["secret"]), g["amount"], g["label"],
               [int(x) for x in g["siblings"]], g["path_bits"], int(g["change_nullifier"]), int(g["change_secret"]), g["excl_low"],
               g["excl_next"], [int(x) for x in g["excl_siblings"]], g["excl_path_bits"])


def test_labeled_golden_proof_reproduced_by_c_port():
    g = GOLD
    cs = lc.build_r1cs(g["depth"])
    pkb, vkb = cport.setup_bytes(cs, *[int(x) for x in g["toxic"]])
    assert hashlib.sha256(pkb["a"] + pkb["b1"] + pkb["b2"] + pkb["l"] + pkb["h"]).hexdigest() == g["pk_queries_sha256"]
    v = g["vk"]
    assert (vkb["alpha1"] + vkb["beta2"] + vkb["gamma2"] + vkb["delta2"] + vkb["ic"]).hex() == v["alpha1"] + v["beta2"] + v["gamma2"] + v["delta2"] + v["ic"]
    w = spec_witness(golden_row(g))
    assert cs.is_satisfied(w)
    assert w[lc.V_XROOT] == xc.BlocklistTree(g["depth"], g["flagged"]).root()
    wit = cport.frs(w)
    assert hashlib.sha256(wit).hexdigest() == g["witness_sha256"]
    assert cport.unfr(wit[32:32 * 8]) == [int(x) for x in g["public"]]
    assert cport.Prover(cs, pkb).prove(wit, int(g["r"]), int(g["s"])).hex() == g["proof"]
    assert ob.verify(vk_blob(vkb, 7), wit[32:32 * 8], bytes.fromhex(g["proof"]))


def test_labels_are_validated_at_the_boundary():
    assert bytes(api._label_array([0, 1, (1 << 32) - 1])) == struct.pack("<3I", 0, 1, (1 << 32) - 1)
    for bad in ([1 << 32], [-1]):
        with pytest.raises(ValueError):
            api._label_array(bad)


# ---- GPU -----------------------------------------------------------------------------------------------------------------
_KEYS = {}


def labeled_keys(ctx, depth):
    """(pk, vk, r1cs, oracle pk bytes, oracle vk bytes) of the depth-`depth` labeled statement, made once per process."""
    if depth not in _KEYS:
        rng = random.Random(90 + depth)
        tw = [rng.randrange(1, R) for _ in range(5)]
        pk, vk = ob.setup_labeled(ctx, depth, *tw)
        cs = lc.build_r1cs(depth)
        pkb, vkb = cport.setup_bytes(cs, *tw)
        _KEYS[depth] = (pk, vk, cs, pkb, vkb)
    return _KEYS[depth]


def proofs_verify(vk, proofs, pub, batch):
    return [ob.verify(vk, pub[224 * i:224 * i + 224], proofs[256 * i:256 * i + 256]) for i in range(batch)]


@pytest.mark.gpu
def test_labeled_hashes_match_oracle(ctx):
    rng = random.Random(91)
    n = 40
    nul = [0, R - 1] + [rng.randrange(R) for _ in range(n - 2)]
    sec = [R - 1, 0] + [rng.randrange(R) for _ in range(n - 2)]
    pre = ctx.labeled_precommitments(cport.frs(nul), cport.frs(sec))
    assert cport.unfr(pre) == [lc.precommitment(a, b) for a, b in zip(nul, sec)]
    tokens = [rng.randrange(R) for _ in range(n)]
    amounts = [0, U64, 1] + [rng.randrange(1 << 64) for _ in range(n - 3)]
    labels = [(1 << 32) - 1, 0, 7] + [rng.randrange(1 << 32) for _ in range(n - 3)]
    leaves = ctx.labeled_leaves(pre, cport.frs(tokens), amounts, labels)
    assert cport.unfr(leaves) == [lc.leaf(p, t, a, l) for p, t, a, l in zip(cport.unfr(pre), tokens, amounts, labels)]
    # uint64 / uint32 buffers are taken as they are
    assert ctx.labeled_leaves(pre, cport.frs(tokens), struct.pack(f"<{n}Q", *amounts), struct.pack(f"<{n}I", *labels)) == leaves
    bad = R.to_bytes(32, "little")
    for args in ((bad + cport.frs(nul[1:2]), cport.frs(sec[:2])), (cport.frs(nul[:2]), cport.frs(sec[:1]) + bad)):
        with pytest.raises(ob.OwshenB200Error) as e:
            ctx.labeled_precommitments(*args)
        assert e.value.code == -4 or "encoding" in str(e.value).lower()
    with pytest.raises(ob.OwshenB200Error):
        ctx.labeled_leaves(bad + pre[32:64], cport.frs(tokens[:2]), amounts[:2], labels[:2])
    with pytest.raises(ob.OwshenB200Error):
        ctx.labeled_leaves(pre[:64], cport.frs(tokens[:1]) + bad, amounts[:2], labels[:2])
    for args in ((pre[:64], cport.frs(tokens[:1]), amounts[:2], labels[:2]), (pre[:64], cport.frs(tokens[:2]), amounts[:1], labels[:2]),
                 (pre[:64], cport.frs(tokens[:2]), amounts[:2], labels[:3]), (pre[:64], cport.frs(tokens[:2]), amounts[:2], [1 << 32, 0])):
        with pytest.raises(ValueError):
            ctx.labeled_leaves(*args)


@pytest.mark.gpu
def test_labeled_witness_matches_oracle(ctx):
    rng = random.Random(92)
    # depth 2: 40 rows with every edge row, the soundness mutations' rows and random inputs anywhere in their types
    bl = xc.BlocklistTree(2, [1, 2])
    good = note_row(rng, 2, 3, bl, amount=1000, withdrawn=300)
    mutated = [note_row(rng, 2, 1, bl, leaf=0), note_row(rng, 2, 1, bl, leaf=1), note_row(rng, 2, 3, bl, leaf=0),
               note_row(rng, 2, 0, bl, leaf=2), dict(good, withdrawn=1001), dict(good, amount=0, withdrawn=U64),
               dict(good, amount=U64, withdrawn=0), dict(good, amount=5, withdrawn=U64), dict(good, label=(1 << 32) - 1),
               dict(good, low=good["next"], next=good["low"]), dict(good, low=U64, next=0), dict(good, low=0, next=U64)]
    rows = edge_rows(rng, 2) + mutated
    rows += valid_rows(rng, 6, 2)
    rows += random_rows(rng, 40 - len(rows), 2)
    assert len(rows) == 40
    assert ctx.labeled_witness(2, *pack(rows)) == oracle_witnesses(rows)
    rows = edge_rows(rng, 32)[:4] + random_rows(rng, 2, 32)
    assert ctx.labeled_witness(32, *pack(rows)) == oracle_witnesses(rows)
    # a field input >= r in any of the eight field arrays
    rows = valid_rows(rng, 2, 2)
    for k in (0, 1, 3, 4, 7, 9, 10, 13):
        p = list(pack(rows))
        p[k] = R.to_bytes(32, "little") + p[k][32:]
        with pytest.raises(ob.OwshenB200Error) as e:
            ctx.labeled_witness(2, *p)
        assert e.value.code == -4 or "encoding" in str(e.value).lower(), k
    # wrong lengths and out-of-range integers
    p = pack(rows)
    for k, bad in ((2, p[2][:1]), (5, p[5] + [0]), (6, p[6][:1]), (6, [1 << 32, 0]), (7, p[7][:-32]), (8, p[8] + [0]), (11, [1 << 64, 0]),
                   (13, p[13] + bytes(32)), (14, p[14][:1])):
        q = list(p)
        q[k] = bad
        with pytest.raises(ValueError):
            ctx.labeled_witness(2, *q)


@pytest.mark.gpu
def test_setup_labeled_matches_oracle(ctx):
    for depth in (2, 32):
        pk, vk, cs, pkb, vkb = labeled_keys(ctx, depth)
        assert pk == pk_blob(cs, pkb, 0), depth
        assert vk == vk_blob(vkb, 7), depth


@pytest.mark.gpu
def test_labeled_key_from_ceremony(ctx):
    """One phase-1 contribution (t, a, b), then the depth-2 key: before phase 2, gamma = delta = 1 (DESIGN.md section 4b)."""
    rng = random.Random(93)
    t, a, b = (rng.randrange(1, R) for _ in range(3))
    acc0 = ob.ptau_new(ctx, 14)                           # the depth-2 labeled domain is 2^14
    acc1, rec = ob.ptau_contribute(ctx, acc0, [t, a, b], [rng.randrange(1, R) for _ in range(3)])
    assert ob.ptau_verify(ctx, acc0, acc1, rec)
    pk, vk = ob.ptau_prepare_labeled(ctx, acc1, 2)
    assert (pk, vk) == ob.setup_labeled(ctx, 2, t, a, b, 1, 1)
    cs = lc.build_r1cs(2)
    pkb, vkb = cport.setup_bytes(cs, t, a, b, 1, 1)
    assert pk == pk_blob(cs, pkb, 0) and vk == vk_blob(vkb, 7)
    PK = ob.ProvingKey(ctx, pk)
    try:
        assert (PK.labeled_depth, PK.exclusion_depth, PK.transfer_depth) == (2, None, None)
    finally:
        PK.close()


@pytest.mark.gpu
@pytest.mark.parametrize("depth,batch", [(2, 40), (32, 3)])
def test_prove_labeled_matches_oracle(ctx, monkeypatch, depth, batch):
    """Default settings, then chunks of 3 on two lanes (a batch above the chunk): both byte for byte the oracle C prover's."""
    pk, vk, cs, pkb, vkb = labeled_keys(ctx, depth)
    rng = random.Random(94 + depth)
    rows = (edge_rows(rng, depth) + valid_rows(rng, batch, depth))[:batch]
    rs = cport.frs([rng.randrange(R) for _ in range(2 * batch)])
    wit = oracle_witnesses(rows)
    exp = cport.Prover(cs, pkb).prove_batch(wit, rs)
    results = []
    for env in (dict(), dict(OG_CHUNK=3 if depth == 2 else 2, OG_LANES=2)):
        set_env(monkeypatch, **env)
        PK = ob.ProvingKey(ctx, pk)
        try:
            assert (PK.n_vars, PK.n_pub, PK.depth, PK.labeled_depth, PK.exclusion_depth) == (cs.n_vars, 7, 0, depth, None)
            results.append(PK.prove_labeled(*pack(rows), rs))
        finally:
            PK.close()
    set_env(monkeypatch)
    nv = cs.n_vars
    for proofs, pub in results:
        assert proofs == exp
        assert pub == b"".join(wit[32 * nv * i + 32:32 * nv * i + 32 * 8] for i in range(batch))
    proofs, pub = results[0]
    assert all(proofs_verify(vk, proofs, pub, batch))
    for k in (3, 5, 6):                                   # another exclusion root, withdrawn or change commitment
        bad = bytearray(pub[:224]); bad[32 * k] ^= 1
        assert not ob.verify(vk, bytes(bad), proofs[:256]), k


@pytest.mark.gpu
def test_prove_labeled_dev_matches_host_entry_point(ctx):
    import torch
    pk = labeled_keys(ctx, 2)[0]
    rng = random.Random(95)
    batch = 5
    rows = valid_rows(rng, batch, 2)
    rs = cport.frs([rng.randrange(R) for _ in range(2 * batch)])
    p = pack(rows)
    PK = ob.ProvingKey(ctx, pk)
    try:
        proofs, pub = PK.prove_labeled(*p, rs)
        fmt = {2: "Q", 5: "Q", 6: "I", 8: "I", 11: "Q", 12: "Q", 14: "I"}
        raw = [struct.pack(f"<{len(x)}{fmt[k]}", *x) if k in fmt else x for k, x in enumerate(p)]
        dev = lambda b: torch.frombuffer(bytearray(b), dtype=torch.uint8).to("cuda")
        d_in = [dev(x) for x in raw + [rs]]
        d_pr = torch.zeros(256 * batch, dtype=torch.uint8, device="cuda")
        d_pub = torch.zeros(224 * batch, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        rc = api.lib().og_groth16_prove_labeled_dev(ctx._h, PK._h, *[api._ptr(t) for t in d_in[:15]], batch, api._ptr(d_in[15]),
                                                    api._ptr(d_pr), api._ptr(d_pub))
        assert rc == 0
        ctx.sync()
        assert bytes(d_pr.cpu().numpy()) == proofs and bytes(d_pub.cpu().numpy()) == pub
    finally:
        PK.close()


@pytest.mark.gpu
def test_labeled_golden_proof(ctx):
    g = GOLD
    pk, vk = ob.setup_labeled(ctx, g["depth"], *[int(x) for x in g["toxic"]])
    v = g["vk"]
    assert vk[12:].hex() == v["alpha1"] + v["beta2"] + v["gamma2"] + v["delta2"] + v["ic"]
    rs = bn.fr_to_bytes(int(g["r"])) + bn.fr_to_bytes(int(g["s"]))
    PK = ob.ProvingKey(ctx, pk)
    try:
        proofs, pub = PK.prove_labeled(*pack([golden_row(g)]), rs)
    finally:
        PK.close()
    assert proofs.hex() == g["proof"]
    assert cport.unfr(pub) == [int(x) for x in g["public"]]
    assert ob.verify(vk, pub, proofs)


# every statement's prover: (name, number of input arrays)
_PROVERS = (("withdraw", 5), ("deposit", 3), ("transfer", 11), ("association", 7), ("exclusion", 9), ("labeled", 15))


@pytest.mark.gpu
def test_six_provers_refuse_each_others_keys(ctx):
    import torch
    d_buf = torch.zeros(1 << 16, dtype=torch.uint8, device="cuda")
    d = api._ptr(d_buf)                                   # every device argument of the _dev entry points
    h = bytes(1 << 16)                                    # every host input of the host entry points
    rng = random.Random(96)
    tw = [rng.randrange(1, R) for _ in range(5)]
    keys = {"withdraw": ob.setup_withdraw(ctx, 2, *tw)[0], "deposit": ob.setup_deposit(ctx, *tw)[0],
            "transfer": ob.setup_transfer(ctx, 2, *tw)[0], "association": ob.setup_association(ctx, 2, *tw)[0],
            "exclusion": ob.setup_exclusion(ctx, 2, *tw)[0], "labeled": labeled_keys(ctx, 2)[0]}
    for owner, pk in keys.items():
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
            if owner != "labeled":
                with pytest.raises(ob.OwshenB200Error):
                    PK.prove_labeled(*pack(valid_rows(rng, 1, 2)), bytes(64))
        finally:
            PK.close()
    PK = ob.ProvingKey(ctx, keys["labeled"])
    try:
        rows = valid_rows(rng, 2, 2)
        assert len(PK.prove_labeled(*pack(rows), cport.frs([rng.randrange(R) for _ in range(4)]))[0]) == 512   # still usable
    finally:
        PK.close()


@pytest.mark.gpu
def test_labeled_deposits_withdrawals_and_blocklists_chain(ctx):
    """Labeled deposits interleaved with plain ones in one depth-32 pool tree; a provider flags one deposit; another is
    withdrawn in part and its change note appended; the change note withdraws again under the same blocklist and leaves a
    second change note.  Once the provider also flags the original deposit, that second change note gets no exclusion
    witness, and a forced neighbouring bracket gives a proof that fails verification: the label carries the flag through
    every note the deposit became."""
    rng = random.Random(97)
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
    flagged_a, b = labels[0], 1                            # the provider flags deposit A; note B withdraws
    xs1 = ob.ExclusionSet(ctx, depth, [flagged_a, 1 << 20])
    pk, vk = labeled_keys(ctx, depth)[:2]
    PK = ob.ProvingKey(ctx, pk)

    def withdraw(nullifier, secret, amount, index, withdrawn, blocklist, low=None, nxt=None, xsibs=None, xbits=None):
        """One labeled withdrawal of the note at pool leaf `index` with label labels[b] -> (change note, public inputs, ok)."""
        if low is None:
            low, nxt, xsibs, xbits = blocklist.witness([labels[b]])
        sibs, bits = pool.paths([index])
        change = (rng.randrange(R), rng.randrange(R), amount - withdrawn)
        recipient = rng.randrange(1 << 160)
        proofs, pub = PK.prove_labeled(cport.frs([token]), cport.frs([recipient]), [withdrawn], cport.frs([nullifier]),
                                       cport.frs([secret]), [amount], [labels[b]], sibs, bits, cport.frs([change[0]]),
                                       cport.frs([change[1]]), low, nxt, xsibs, xbits, cport.frs([rng.randrange(R), rng.randrange(R)]))
        p = cport.unfr(pub)
        assert p[:6] == [as_int(pool.root()), mimc7.multi_hash([nullifier], key=1), recipient, as_int(blocklist.root()), token, withdrawn]
        assert p[6] == lc.leaf(lc.precommitment(change[0], change[1]), token, change[2], labels[b])
        return change, pub, ob.verify(vk, pub, proofs)

    try:
        with pytest.raises(ValueError, match=str(flagged_a)):
            xs1.witness([flagged_a])
        # a partial withdrawal of deposit B; the node appends its change commitment
        nb = notes[b]
        change1, pub, ok = withdraw(nb[0], nb[1], nb[2], labels[b], nb[2] // 3, xs1)
        assert ok
        i1 = pool.insert(pub[32 * 6:32 * 7])
        plain(1)
        # the change note withdraws again under the same blocklist, at its own index and with B's label
        change2, pub, ok = withdraw(change1[0], change1[1], change1[2], i1, 12345, xs1)
        assert ok
        i2 = pool.insert(pub[32 * 6:32 * 7])
        # the provider's next version also flags deposit B: no witness for B's label, and the neighbouring brackets fail
        xs2 = ob.ExclusionSet(ctx, depth, [flagged_a, labels[b], 1 << 20])
        with pytest.raises(ValueError, match=str(labels[b])):
            xs2.witness([labels[b]])
        j_b = xs2.keys.index(labels[b] + 1)
        for j in (j_b - 1, j_b):                                # the leaves (k_j, B + 1) and (B + 1, k_j+2)
            xsibs, xbits = xs2.tree.paths([j])
            _, _, ok = withdraw(change2[0], change2[1], change2[2], i2, 1, xs2, [xs2.keys[j]], [xs2.keys[j + 1]], xsibs, xbits)
            assert not ok, j
        # under the old version the same note still withdraws
        assert withdraw(change2[0], change2[1], change2[2], i2, 1, xs1)[2]
    finally:
        PK.close()
