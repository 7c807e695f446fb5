"""The ragequit statement (oracle/ragequit_circuit.py == csrc/withdraw_circuit.hpp: RagequitBuilder): the spec, its soundness
mutations and domain separation, the R1CS export, the envelope, the GPU witness, setup and batched prover against the oracle,
ten-way key refusal, and a depth-32 chain of owned labeled deposits, ragequits and an approved transfer through one pool
tree, one ApprovedLabels set and one nullifier set."""
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
from oracle import labeled_circuit as lc
from oracle import owned_circuit as oc
from oracle import owned_labeled_circuit as olc
from oracle import ragequit_circuit as rqc
from oracle import withdraw_circuit as wc
from tests.helpers import pk_blob, vk_blob

R = bn.R
U64, U32 = (1 << 64) - 1, (1 << 32) - 1
OG_E_ENCODING = -2             # include/owshen_b200.h: a non-canonical field element
GOLD = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "ragequit_vectors.json")))
STATEMENTS = ("withdraw", "deposit", "transfer", "association", "exclusion", "labeled", "labeled_association", "owned_transfer",
              "owned_labeled_transfer", "ragequit")
_PROVERS = (("withdraw", 5), ("deposit", 3), ("transfer", 11), ("association", 7), ("exclusion", 9), ("labeled", 15),
            ("labeled_association", 13), ("owned_transfer", 11), ("owned_labeled_transfer", 15), ("ragequit", 9))
fr = lambda xs: b"".join(x.to_bytes(32, "little") for x in xs)
word_of = lambda bits: sum(b << l for l, b in enumerate(bits))


# ---- rows: one ragequit's inputs as ints ---------------------------------------------------------------------------------
def row(root, token, amount, label, recipient, spend_key, blinding, sibs, bits):
    return (root, token, amount, label, recipient, spend_key, blinding, sibs, bits)


def opened(tree, i):
    sibs, bits = tree.path(i)
    return sibs, word_of(bits)


def deposit_tree(rng, depth, notes, before=1):
    """A spec pool tree with `before` random leaves, then one owned labeled deposit per (spend_key, blinding, token, amount),
    each labelled with its own leaf index -> (tree, labels)."""
    tree = mimc7.MerkleTree(depth)
    for _ in range(before):
        tree.insert(rng.randrange(R))
    labels = []
    for s, b, tok, am in notes:
        labels.append(tree.insert(olc.note_leaf(olc.spend_public_key(s), b, tok, am, tree.n_leaves)))
    return tree, labels


def valid_rows(rng, batch, depth):
    """Rows that satisfy the statement: each ragequits the deposit at a random index of its own tree."""
    rows = []
    for _ in range(batch):
        s, b, tok, am = rng.randrange(R), rng.randrange(R), rng.randrange(R), rng.randrange(1 << 64)
        tree, (la,) = deposit_tree(rng, depth, [(s, b, tok, am)], before=rng.randrange(min(1 << depth, 8)))
        sibs, bits = opened(tree, la)
        rows.append(row(tree.root(), tok, am, la, rng.randrange(1 << 160), s, b, sibs, bits))
    return rows


def random_rows(rng, batch, depth):
    """Rows of uniformly random inputs, path bits above `depth` set (their witnesses do not satisfy the statement: the
    witness kernel does not care)."""
    high = 0 if depth == 32 else (U32 >> depth) << depth
    return [row(rng.randrange(R), rng.randrange(R), rng.randrange(1 << 64), rng.randrange(1 << 32), rng.randrange(R),
                rng.randrange(R), rng.randrange(R), [rng.randrange(R) for _ in range(depth)], rng.randrange(1 << 32) | high)
            for _ in range(batch)]


def pack(rows):
    """The nine input buffers of og_ragequit_witness / og_groth16_prove_ragequit."""
    f = cport.frs
    return (f([r[0] for r in rows]), f([r[1] for r in rows]), f([r[4] for r in rows]), struct.pack(f"<{len(rows)}Q", *[r[2] for r in rows]),
            [r[3] for r in rows], f([r[5] for r in rows]), f([r[6] for r in rows]), f([s for r in rows for s in r[7]]), [r[8] for r in rows])


def oracle_witnesses(rows):
    return b"".join(cport.frs(rqc.witness(*r)) for r in rows)


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
def test_ragequit_sizes():
    for depth in (1, 2, 32):
        L = rqc.Layout(depth)
        P = L.perm
        assert (L.n_vars, L.n_constraints) == (12 + 10 * P + depth * (2 * P + 4), 5 + 10 * P + depth * (2 * P + 3))
    expect = {1: (4384, 4376, 13), 2: (5116, 5107, 13), 32: (27076, 27037, 15)}
    for depth, (nv, nc, log_m) in expect.items():
        cs = rqc.build_r1cs(depth)
        assert (cs.n_vars, cs.n_constraints, cs.n_pub) == (nv, nc, 6), depth
        assert g16.domain_log(cs.n_constraints, cs.n_pub) == log_m, depth
        assert ob.ragequit_r1cs_info(depth) == dict(n_constraints=nc, n_vars=nv, n_pub=6, log_m=log_m), depth
    for bad in (0, 33):
        with pytest.raises(ob.OwshenB200Error):
            ob.ragequit_r1cs_info(bad)


def test_ten_statement_shapes_are_distinct():
    """The prover recognises a key by (n_pub, n_vars, n_constraints) and ProvingKey by (n_vars, n_pub): no two (statement,
    depth) pairs of the ten share either."""
    seen = {}
    for stmt in STATEMENTS:
        for d in (range(1, 33) if stmt != "deposit" else (0,)):
            i = api._statement_r1cs_info(stmt, d)
            shape = (i["n_pub"], i["n_vars"], i["n_constraints"])
            assert shape not in seen, (stmt, d, seen.get(shape))
            assert (shape[0], shape[1]) not in {(s[0], s[1]) for s in seen}, (stmt, d)
            seen[shape] = (stmt, d)
    assert [s[0] for s in seen].count(6) == 32                # n_pub = 6: this statement alone
    assert {seen[s][0] for s in seen if s[0] == 6} == {"ragequit"}


def test_ragequit_r1cs_export_matches_spec():
    for depth in (1, 2, 32):
        cs = rqc.build_r1cs(depth)
        for m in "ABC":
            assert ob.ragequit_r1cs_export(depth, m) == cs.csr(m), (depth, m)


@pytest.fixture(scope="module")
def cs2():
    return rqc.build_r1cs(2)


def test_ragequit_witnesses_satisfy(cs2):
    rng = random.Random(500)
    tok = rng.randrange(1 << 160)
    # the deposit leaf itself: index = label
    s, b = rng.randrange(R), rng.randrange(R)
    tree, (la,) = deposit_tree(rng, 2, [(s, b, tok, 77)], before=2)
    assert la == 2
    w = rqc.witness(tree.root(), tok, 77, la, 5, s, b, *opened(tree, la))
    assert cs2.is_satisfied(w)
    assert w[1:7] == [tree.root(), tok, 77, la, 5, olc.nullifier(s, olc.note_leaf(olc.spend_public_key(s), b, tok, 77, la), la)]
    # a transfer output under label 0 at index 3
    tree = mimc7.MerkleTree(2)
    for _ in range(3):
        tree.insert(rng.randrange(R))
    i = tree.insert(olc.note_leaf(olc.spend_public_key(s), b, tok, 40, 0))
    assert i == 3 and cs2.is_satisfied(rqc.witness(tree.root(), tok, 40, 0, 5, s, b, *opened(tree, i)))
    # amounts 0 and 2^64 - 1, labels 0 and 2^32 - 1, leaf indices 0 and 2^depth - 1
    for am in (0, U64):
        for la in (0, U32):
            for idx in (0, 3):
                tree = mimc7.MerkleTree(2)
                for _ in range(idx):
                    tree.insert(rng.randrange(R))
                tree.insert(olc.note_leaf(olc.spend_public_key(s), b, tok, am, la))
                w = rqc.witness(tree.root(), tok, am, la, rng.randrange(1 << 160), s, b, *opened(tree, idx))
                assert cs2.is_satisfied(w), (am, la, idx)
                assert (w[rqc.V_AMOUNT], w[rqc.V_LABEL]) == (am, la)
    # one note at two leaves: two different nullifiers, both valid
    tree = mimc7.MerkleTree(2)
    lf = olc.note_leaf(olc.spend_public_key(s), b, tok, 9, 1)
    i0, i1 = tree.insert(lf), tree.insert(lf)
    w0, w1 = (rqc.witness(tree.root(), tok, 9, 1, 5, s, b, *opened(tree, i)) for i in (i0, i1))
    assert cs2.is_satisfied(w0) and cs2.is_satisfied(w1) and w0[rqc.V_NF] != w1[rqc.V_NF]
    # only the low depth bits of the path word count
    sibs, bits = opened(tree, i1)
    assert rqc.witness(tree.root(), tok, 9, 1, 5, s, b, sibs, bits | 0xFFFFFFF0) == w1


def test_ragequit_mutations_fail_named_rows(cs2):
    rng = random.Random(501)
    L = rqc.Layout(2)
    s, b, tok, am = rng.randrange(R), rng.randrange(R), rng.randrange(1 << 160), 1234
    tree, (la,) = deposit_tree(rng, 2, [(s, b, tok, am)])
    sibs, bits = opened(tree, la)
    root, P = tree.root(), olc.spend_public_key(s)
    base = rqc.witness(root, tok, am, la, 99, s, b, sibs, bits)
    assert cs2.is_satisfied(base)
    # a wrong spend key, and the sender's guesses (P, the blinding): owner, leaf and path are consistent but reach another root
    for guess in ((s + 1) % R, P, b, 0, R - 1):
        assert failing(cs2, rqc.witness(root, tok, am, la, 99, guess, b, sibs, bits)) == [L.row_root], guess
    # a tampered amount, label or token: the leaf is another leaf
    for am2, la2, tok2 in ((am + 1, la, tok), (U64, la, tok), (am, la + 1, tok), (am, 0, tok), (am, la, tok + 1)):
        assert failing(cs2, rqc.witness(root, tok2, am2, la2, 99, s, b, sibs, bits)) == [L.row_root], (am2, la2, tok2)
    # a wrong blinding, and a wrong path bit
    assert failing(cs2, rqc.witness(root, tok, am, la, 99, s, b + 1, sibs, bits)) == [L.row_root]
    for flip in (1, 2):
        assert failing(cs2, rqc.witness(root, tok, am, la, 99, s, b, sibs, bits ^ flip)) == [L.row_root], flip
    # a tampered nullifier
    w = list(base)
    w[rqc.V_NF] = (w[rqc.V_NF] + 1) % R
    assert failing(cs2, w) == [L.row_nf]
    # the nullifier of another index (the leaf's, computed honestly) does not bind either
    w = list(base)
    w[rqc.V_NF] = olc.nullifier(s, olc.note_leaf(P, b, tok, am, la), la ^ 1)
    assert failing(cs2, w) == [L.row_nf]
    # a tampered recipient^2
    w = list(base)
    w[rqc.V_RSQ] = (w[rqc.V_RSQ] + 1) % R
    assert failing(cs2, w) == [0]
    # a zero-value note off the tree: the root row is unconditional
    assert failing(cs2, rqc.witness(root, tok, 0, la, 99, s, b, sibs, bits)) == [L.row_root]


def test_domain_separation_and_the_shared_nullifier():
    rng = random.Random(502)
    cs2 = rqc.build_r1cs(2)
    L = rqc.Layout(2)
    s, b, tok, am, la = rng.randrange(R), rng.randrange(R), rng.randrange(1 << 160), 50, 1
    P = olc.spend_public_key(s)
    pre = olc.precommitment(P, b)
    # key-0, key-2 and key-4 leaves over the same words, and the families' own leaves of the note: none opens here
    foreign = [mimc7.multi_hash([pre, tok, am, la], key=k) for k in (0, 2, 4)]
    foreign += [lc.leaf(lc.precommitment(P, b), tok, am, la), oc.commitment(P, b, tok, am), mimc7.multi_hash([P, b, tok, am], key=0)]
    for f in foreign:
        tree = mimc7.MerkleTree(2)
        tree.insert(rng.randrange(R))
        i = tree.insert(f)
        assert failing(cs2, rqc.witness(tree.root(), tok, am, la, 1, s, b, *opened(tree, i))) == [L.row_root]
    # the ragequit nullifier of a note is input 0's nullifier in an owned labeled transfer of the same note
    tree = mimc7.MerkleTree(2)
    tree.insert(rng.randrange(R))
    i = tree.insert(olc.leaf(pre, tok, am, la))
    sibs, bits = opened(tree, i)
    w = rqc.witness(tree.root(), tok, am, la, 1, s, b, sibs, bits)
    assert cs2.is_satisfied(w)
    dummy = (rng.randrange(R), rng.randrange(R), 0, [0, 0], 0)
    wt = olc.witness(tree.root(), tok, 0, 1, la, [(s, b, am, sibs, bits), dummy], [(P, 1, am), (P, 2, 0)], [0, 0], 0)
    assert w[rqc.V_NF] == wt[olc.V_NF[0]] == oc.nullifier(s, olc.leaf(pre, tok, am, la), i)


def golden_row(g):
    return row(int(g["root"]), int(g["token"]), int(g["amount"]), int(g["label"]), int(g["recipient"]), int(g["spend_key"]),
               int(g["blinding"]), [int(x) for x in g["siblings"]], int(g["path_bits"]))


def test_ragequit_golden_proof_reproduced_by_c_port():
    g = GOLD
    cs = rqc.build_r1cs(g["depth"])
    pkb, vkb = cport.setup_bytes(cs, *[int(x) for x in g["toxic"]])
    assert hashlib.sha256(pkb["a"] + pkb["b1"] + pkb["b2"] + pkb["l"] + pkb["h"]).hexdigest() == g["pk_queries_sha256"]
    w = rqc.witness(*golden_row(g))
    assert cs.is_satisfied(w)
    wit = cport.frs(w)
    assert hashlib.sha256(wit).hexdigest() == g["witness_sha256"]
    assert cport.unfr(wit[32:32 * 7]) == [int(x) for x in g["public"]]
    assert cport.Prover(cs, pkb).prove(wit, int(g["r"]), int(g["s"])).hex() == g["proof"]
    assert ob.verify(vk_blob(vkb, 6), wit[32:32 * 7], bytes.fromhex(g["proof"]))


def test_ragequit_envelope():
    rng = random.Random(503)
    proof, pub = bytes(rng.randrange(256) for _ in range(256)), fr([rng.randrange(R) for _ in range(6)])
    msg = formats.shielded_ragequit_to_rlp(proof, pub)
    assert formats.shielded_ragequit_from_rlp(msg) == (proof, pub)
    words = [pub[32 * i:32 * i + 32] for i in range(6)]
    bad = [formats.rlp_encode(["shielded-withdraw", proof] + words),                    # a wrong kind
           formats.rlp_encode(["shielded-labeled-transfer", proof] + words),
           formats.rlp_encode(["shielded-ragequit", proof[:255]] + words),               # a wrong length
           formats.rlp_encode(["shielded-ragequit", proof] + words[:5] + [words[5] + b"\x00"]),
           formats.rlp_encode(["shielded-ragequit", proof] + words[:5]),                 # a wrong count
           formats.rlp_encode(["shielded-ragequit", proof] + words + [words[0]]),
           formats.rlp_encode(["shielded-ragequit", proof] + words[:5] + [[words[5]]]),
           msg + b"\x00"]
    for m in bad:
        with pytest.raises(ValueError):
            formats.shielded_ragequit_from_rlp(m)
    with pytest.raises(ValueError):
        formats.shielded_withdraw_from_rlp(msg)
    for p, q in ((proof[:255], pub), (proof, pub[:160]), (proof, pub + bytes(32))):
        with pytest.raises(ValueError):
            formats.shielded_ragequit_to_rlp(p, q)


# ---- GPU -----------------------------------------------------------------------------------------------------------------
_KEYS = {}


def keys(ctx, depth):
    """(pk, vk, r1cs, oracle pk bytes, oracle vk bytes) of the depth-`depth` ragequit statement, once per process."""
    if depth not in _KEYS:
        rng = random.Random(510 + depth)
        tw = [rng.randrange(1, R) for _ in range(5)]
        pk, vk = ob.setup_ragequit(ctx, depth, *tw)
        cs = rqc.build_r1cs(depth)
        pkb, vkb = cport.setup_bytes(cs, *tw)
        _KEYS[depth] = (pk, vk, cs, pkb, vkb)
    return _KEYS[depth]


def proofs_verify(vk, proofs, pub, batch):
    return [ob.verify(vk, pub[192 * i:192 * i + 192], proofs[256 * i:256 * i + 256]) for i in range(batch)]


@pytest.mark.gpu
def test_ragequit_witness_matches_oracle(ctx):
    rng = random.Random(504)
    for depth in (2, 32):
        rows = random_rows(rng, 37 if depth == 2 else 5, depth) + valid_rows(rng, 3, depth)
        assert ctx.ragequit_witness(depth, *pack(rows)) == oracle_witnesses(rows), depth
    # edge values: amounts 0 and 2^64 - 1, labels 0 and 2^32 - 1, field inputs 0 and r - 1
    rows = [row(x, x, a, la, x, x, x, [x, x], 0xFFFFFFFF) for a, la in ((0, 0), (U64, U32), (1, 7)) for x in (0, R - 1)]
    assert ctx.ragequit_witness(2, *pack(rows)) == oracle_witnesses(rows)
    for k in (0, 1, 2, 5, 6, 7):                          # a field input >= r
        p = list(pack(rows[:1]))
        p[k] = R.to_bytes(32, "little") + p[k][32:]
        with pytest.raises(ob.OwshenB200Error) as e:
            ctx.ragequit_witness(2, *p)
        assert e.value.code == OG_E_ENCODING, k
    # the boundary: depth 0 and 33, null pointers, a batch of 0
    bufs = [api._u32_array(x) if isinstance(x, list) else x for x in pack(rows[:1])]
    nv = rqc.Layout(2).n_vars
    out = api.C.create_string_buffer(32 * nv)
    fn = api.lib().og_ragequit_witness
    for d in (0, 33):
        assert fn(ctx._h, d, *[api._ptr(x) for x in bufs], 1, out) == api.OG_E_INVALID, d
    for k in range(9):
        args = [api._ptr(x) for x in bufs]
        args[k] = None
        assert fn(ctx._h, 2, *args, 1, out) == api.OG_E_INVALID, k
    assert fn(ctx._h, 2, *[api._ptr(x) for x in bufs], 1, None) == api.OG_E_INVALID
    assert fn(ctx._h, 2, *[api._ptr(x) for x in bufs], 0, out) == api.OG_OK


@pytest.mark.gpu
def test_setup_ragequit_matches_oracle(ctx):
    for depth in (2, 32):
        pk, vk, cs, pkb, vkb = keys(ctx, depth)
        assert pk == pk_blob(cs, pkb, 0), depth
        assert vk == vk_blob(vkb, 6), depth


@pytest.mark.gpu
def test_ragequit_key_from_ceremony(ctx):
    rng = random.Random(505)
    t, a, b, d = (rng.randrange(1, R) for _ in range(4))
    acc0 = ob.ptau_new(ctx, 13)                           # the depth-2 domain is 2^13
    acc1, rec = ob.ptau_contribute(ctx, acc0, [t, a, b], [rng.randrange(1, R) for _ in range(3)])
    assert ob.ptau_verify(ctx, acc0, acc1, rec)
    pk0, vk0 = ob.ptau_prepare_ragequit(ctx, acc1, 2)
    assert (pk0, vk0) == ob.setup_ragequit(ctx, 2, t, a, b, 1, 1)
    pk, vk, rec2 = ob.phase2_contribute(ctx, pk0, vk0, d, rng.randrange(1, R))
    assert ob.phase2_verify(ctx, pk0, vk0, pk, vk, rec2)
    assert (pk, vk) == ob.setup_ragequit(ctx, 2, t, a, b, 1, d)
    PK = ob.ProvingKey(ctx, pk)
    try:
        assert (PK.ragequit_depth, PK.owned_labeled_transfer_depth) == (2, None)
        rows = valid_rows(rng, 2, 2)
        proofs, pub = PK.prove_ragequit(*pack(rows), cport.frs([rng.randrange(R) for _ in range(4)]))
        assert all(proofs_verify(vk, proofs, pub, 2))
    finally:
        PK.close()


@pytest.mark.gpu
@pytest.mark.parametrize("depth,batch", [(2, 40), (32, 3)])
def test_prove_ragequit_matches_oracle(ctx, monkeypatch, depth, batch):
    """Default settings, then chunks below the batch on one and two lanes: all byte for byte the oracle C prover's."""
    pk, vk, cs, pkb, vkb = keys(ctx, depth)
    rng = random.Random(520 + depth)
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
            assert (PK.n_vars, PK.n_pub, PK.depth, PK.ragequit_depth) == (cs.n_vars, 6, 0, depth)
            results.append(PK.prove_ragequit(*pack(rows), rs))
        finally:
            PK.close()
    set_env(monkeypatch)
    nv = cs.n_vars
    for proofs, pub in results:
        assert proofs == exp
        assert pub == b"".join(wit[32 * nv * i + 32:32 * nv * i + 32 * 7] for i in range(batch))
    proofs, pub = results[0]
    assert all(proofs_verify(vk, proofs, pub, batch))
    bad = bytearray(pub[:192]); bad[32 * 5] ^= 1          # another nullifier
    assert not ob.verify(vk, bytes(bad), proofs[:256])


@pytest.mark.gpu
def test_prove_ragequit_dev_matches_host_entry_point(ctx):
    import torch
    pk = keys(ctx, 2)[0]
    rng = random.Random(506)
    batch = 4
    rows = valid_rows(rng, batch, 2)
    rs = cport.frs([rng.randrange(R) for _ in range(2 * batch)])
    p = pack(rows)
    PK = ob.ProvingKey(ctx, pk)
    try:
        proofs, pub = PK.prove_ragequit(*p, rs)
        u32 = lambda xs: struct.pack(f"<{len(xs)}I", *xs)
        host = [u32(x) if isinstance(x, list) else x for x in p]
        dev = lambda b: torch.frombuffer(bytearray(b), dtype=torch.uint8).to("cuda")
        d_in = [dev(x) for x in host + [rs]]
        d_pr = torch.zeros(256 * batch, dtype=torch.uint8, device="cuda")
        d_pub = torch.zeros(192 * batch, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        rc = api.lib().og_groth16_prove_ragequit_dev(ctx._h, PK._h, *[api._ptr(t) for t in d_in[:9]], batch, api._ptr(d_in[9]),
                                                     api._ptr(d_pr), api._ptr(d_pub))
        assert rc == 0
        ctx.sync()
        assert bytes(d_pr.cpu().numpy()) == proofs and bytes(d_pub.cpu().numpy()) == pub
    finally:
        PK.close()


@pytest.mark.gpu
def test_ragequit_golden_proof(ctx):
    g = GOLD
    pk, vk = ob.setup_ragequit(ctx, g["depth"], *[int(x) for x in g["toxic"]])
    v = g["vk"]
    assert vk[12:].hex() == v["alpha1"] + v["beta2"] + v["gamma2"] + v["delta2"] + v["ic"]
    rs = bn.fr_to_bytes(int(g["r"])) + bn.fr_to_bytes(int(g["s"]))
    PK = ob.ProvingKey(ctx, pk)
    try:
        proofs, pub = PK.prove_ragequit(*pack([golden_row(g)]), rs)
    finally:
        PK.close()
    assert proofs.hex() == g["proof"]
    assert cport.unfr(pub) == [int(x) for x in g["public"]]
    assert ob.verify(vk, pub, proofs)


@pytest.mark.gpu
def test_ten_provers_refuse_each_others_keys(ctx):
    import torch
    d_buf = torch.zeros(1 << 16, dtype=torch.uint8, device="cuda")
    d = api._ptr(d_buf)                                   # every device argument of the _dev entry points
    h = bytes(1 << 16)                                    # every host input of the host entry points
    rng = random.Random(507)
    tw = [rng.randrange(1, R) for _ in range(5)]
    all_keys = {"withdraw": ob.setup_withdraw(ctx, 2, *tw)[0], "deposit": ob.setup_deposit(ctx, *tw)[0],
                "transfer": ob.setup_transfer(ctx, 2, *tw)[0], "association": ob.setup_association(ctx, 2, *tw)[0],
                "exclusion": ob.setup_exclusion(ctx, 2, *tw)[0], "labeled": ob.setup_labeled(ctx, 2, *tw)[0],
                "labeled_association": ob.setup_labeled_association(ctx, 2, *tw)[0],
                "owned_transfer": ob.setup_owned_transfer(ctx, 2, *tw)[0],
                "owned_labeled_transfer": ob.setup_owned_labeled_transfer(ctx, 2, *tw)[0], "ragequit": keys(ctx, 2)[0]}
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
            if owner != "ragequit":
                with pytest.raises(ob.OwshenB200Error):
                    PK.prove_ragequit(*pack(valid_rows(rng, 1, 2)), bytes(64))
        finally:
            PK.close()
    PK = ob.ProvingKey(ctx, all_keys["ragequit"])
    try:
        rows = valid_rows(rng, 2, 2)
        assert len(PK.prove_ragequit(*pack(rows), cport.frs([rng.randrange(R) for _ in range(4)]))[0]) == 512
    finally:
        PK.close()


@pytest.mark.gpu
def test_ragequit_chain(ctx):
    """Through one depth-32 pool tree with plain and labeled leaves between the owned labeled deposits, and one ApprovedLabels
    set that approves some of them: an unapproved deposit ragequits with the nullifier an approved transfer of it would
    publish, B ragequits the note A transferred to B, A cannot ragequit B's note, and altered public inputs do not verify."""
    from owshen_b200 import ApprovedLabels
    pk, vk = keys(ctx, 32)[:2]
    rng = random.Random(508)
    tw = [rng.randrange(1, R) for _ in range(5)]
    tpk, tvk = ob.setup_owned_labeled_transfer(ctx, 32, *tw)
    tree = ob.MerkleTree(ctx, 32)
    tree.insert_batch([rng.randrange(R) for _ in range(3)])
    token = rng.randrange(1 << 160)
    as_int = lambda b: int.from_bytes(b, "little")
    fr1 = lambda x: x.to_bytes(32, "little")
    u64 = lambda x: struct.pack("<Q", x)
    PK, TPK = ob.ProvingKey(ctx, pk), ob.ProvingKey(ctx, tpk)
    try:
        sa, sb = rng.randrange(R), rng.randrange(R)
        Pa, Pb = cport.unfr(ctx.owned_public_keys(fr([sa, sb])))
        # owned labeled deposits of A between plain and labeled leaves
        ba = [rng.randrange(R) for _ in range(3)]
        pre = ctx.owned_labeled_precommitments(fr([Pa] * 3), fr(ba))
        amts = [100, 70, 55]
        la = ob.deposit_owned_labeled(tree, pre[:32], fr1(token), amts[:1])
        l_label = ob.deposit_labeled(tree, ctx.labeled_precommitments(fr([7]), fr([8])), fr1(token), [40])
        tree.insert(rng.randrange(R))
        lb = ob.deposit_owned_labeled(tree, pre[32:], fr([token, token]), amts[1:])
        labels = la + lb
        assert labels == [3, 6, 7] and l_label == [4]
        approved = ApprovedLabels(ctx, 32, [labels[0], l_label[0]])

        def ragequit(s, b, amount, label, index, recipient):
            sib, bits = tree.paths([index])
            proofs, pub = PK.prove_ragequit(tree.root(), fr1(token), fr1(recipient), u64(amount), [label], fr1(s), fr1(b), sib, bits,
                                            cport.frs([rng.randrange(R) for _ in range(2)]))
            r = row(as_int(tree.root()), token, amount, label, recipient, s, b, cport.unfr(sib), bits[0])
            assert pub == cport.frs(rqc.witness(*r)[1:7])
            return proofs, pub

        # 1. the unapproved deposit at label 6 ragequits in public; the proof verifies with its inputs as given
        with pytest.raises(ValueError):
            approved.witness([labels[1]])
        recipient = rng.randrange(1 << 160)
        proofs, pub = ragequit(sa, ba[1], 70, labels[1], labels[1], recipient)
        assert ob.verify(vk, pub, proofs)
        assert cport.unfr(pub[:160]) == [as_int(tree.root()), token, 70, labels[1], recipient]
        assert formats.shielded_ragequit_from_rlp(formats.shielded_ragequit_to_rlp(proofs, pub)) == (proofs, pub)
        # 2. its nullifier is og_owned_nullifiers' of (s, leaf, index)
        leaf6 = olc.note_leaf(Pa, ba[1], token, 70, labels[1])
        nf6 = pub[160:192]
        assert nf6 == ctx.owned_nullifiers(fr1(sa), fr1(leaf6), [labels[1]])
        # 3. once approved, an owned labeled transfer of the same note publishes the same nullifier: one nullifier set
        #    refuses the second spend
        approved.approve([labels[1]])

        def transfer(label, ins, outs):
            asib, abits = approved.witness([label])
            tr = (as_int(tree.root()), token, 0, 0, label, ins, outs, cport.unfr(asib), abits[0])
            f = cport.frs
            arrays = (f([tr[0]]), f([tr[1]]), f([tr[3]]), u64(tr[2]), [label], f([n[0] for n in ins]), f([n[1] for n in ins]),
                      struct.pack("<2Q", *[n[2] for n in ins]), f([x for n in ins for x in n[3]]), [n[4] for n in ins],
                      f([n[0] for n in outs]), f([n[1] for n in outs]), struct.pack("<2Q", *[n[2] for n in outs]), asib, abits)
            proofs, pub = TPK.prove_owned_labeled_transfer(*arrays, cport.frs([rng.randrange(R) for _ in range(2)]))
            assert ob.verify(tvk, pub, proofs)
            return pub

        def spend_in(s, b, a, index):
            sib, bits = tree.paths([index])
            return (s, b, a, cport.unfr(sib), bits[0])

        dummy = (rng.randrange(R), rng.randrange(R), 0, [0] * 32, 0)
        tpub = transfer(labels[1], [spend_in(sa, ba[1], 70, labels[1]), dummy], [(Pa, 1, 70), (Pa, 2, 0)])
        assert tpub[32 * 5:32 * 6] == nf6
        # 4. A transfers deposit 3 (approved) to B; B ragequits that output, at an index that is not its label
        b_out = rng.randrange(R)
        tpub = transfer(labels[0], [spend_in(sa, ba[0], 100, labels[0]), dummy], [(Pb, b_out, 60), (Pa, rng.randrange(R), 40)])
        idx_b = tree.insert(as_int(tpub[32 * 7:32 * 8]))
        tree.insert(as_int(tpub[32 * 8:32 * 9]))
        assert idx_b != labels[0]
        proofs, pub = ragequit(sb, b_out, 60, labels[0], idx_b, recipient)
        assert ob.verify(vk, pub, proofs)
        leaf_b = olc.note_leaf(Pb, b_out, token, 60, labels[0])
        assert pub[160:192] == ctx.owned_nullifiers(fr1(sb), fr1(leaf_b), [idx_b])
        # 5. A knows B's note but not sb: A's own key, P_b or the blinding as spend key fail verification
        for guess in (sa, Pb, b_out):
            proofs, pub = ragequit(guess, b_out, 60, labels[0], idx_b, recipient)
            assert not ob.verify(vk, pub, proofs), guess
        # 6. public inputs altered after proving: the amount or the label
        proofs, pub = ragequit(sa, ba[2], 55, labels[2], labels[2], recipient)
        assert ob.verify(vk, pub, proofs)
        for k, x in ((2, 56), (2, 0), (3, labels[1]), (3, labels[2] + 1)):
            bad = pub[:32 * k] + fr1(x) + pub[32 * k + 32:]
            assert not ob.verify(vk, bad, proofs), (k, x)
    finally:
        PK.close()
        TPK.close()
