"""The exclusion withdraw statement (oracle/exclusion_circuit.py == csrc/withdraw_circuit.hpp: ExclusionBuilder): its spec and
soundness mutations, the library's R1CS export, GPU witness, setup, ceremony key and batched prover against the oracle, the
GPU-built blocklist tree (ExclusionSet), and a deposit -> pool tree + blocklist tree -> withdrawal chain."""
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
from oracle import exclusion_circuit as xc
from oracle import groth16 as g16
from oracle import transfer_circuit as tc
from oracle import withdraw_circuit as wc
from tests.helpers import pk_blob, vk_blob

R = bn.R
GOLD = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "exclusion_vectors.json")))
GIB = 1 << 30
LANE_BUDGET = 28 * GIB          # csrc/groth16.cu: LANE_SCRATCH_BUDGET
P = 4 * mimc7.N_ROUNDS


# ---- rows: one proof's inputs as ints ---------------------------------------------------------------------------------------
def row(nullifier, secret, recipient, sibs, bits, low, next_, xsibs, xbits):
    """bits / xbits: path words, bit l set when the level-l node is a right child; bits is the note's pool leaf index."""
    return dict(nullifier=nullifier, secret=secret, recipient=recipient, sibs=sibs, bits=bits, low=low, next=next_, xsibs=xsibs,
                xbits=xbits)


def bit_list(word, depth):
    return [(word >> l) & 1 for l in range(depth)]


def bit_word(bits):
    return sum(b << l for l, b in enumerate(bits))


def spec_witness(r):
    d = len(r["sibs"])
    return xc.witness(r["nullifier"], r["secret"], r["recipient"], r["sibs"], bit_list(r["bits"], d), r["low"], r["next"], r["xsibs"],
                      bit_list(r["xbits"], d))


def note_row(rng, depth, index, blocklist, leaf=None):
    """A random note at pool leaf `index` (random pool siblings: the pool root is derived) with the blocklist path of `leaf`
    (default: the leaf that brackets the index)."""
    j = blocklist.bracket(index) if leaf is None else leaf
    xsibs, xbits = blocklist.tree.path(j)
    return row(rng.randrange(R), rng.randrange(R), rng.randrange(1 << 160), [rng.randrange(R) for _ in range(depth)], index,
               blocklist.keys[j], blocklist.keys[j + 1], xsibs, bit_word(xbits))


def edge_rows(rng, depth):
    """Satisfying rows at the edges: an empty blocklist, index 0, index 2^depth - 1, a note whose neighbours are both flagged,
    and (depth 2) the one unflagged index of a full tree."""
    top = (1 << depth) - 1
    mid = min(5, top - 1)
    cases = [([], 0), ([], top), ([top], 0), ([0], top), ([mid - 1, mid + 1], mid), ([0, top - 1], top), ([1, top], 0)]
    if depth == 2:
        cases += [([0, 1, 2], 3), ([1, 2, 3], 0), ([0, 1, 3], 2)]
    return [note_row(rng, depth, i, xc.BlocklistTree(depth, flagged)) for flagged, i in cases]


def valid_rows(rng, batch, depth):
    """Rows whose note is unflagged in a random blocklist."""
    rows = []
    for _ in range(batch):
        flagged = sorted(set(rng.randrange(1 << depth) for _ in range(rng.randrange(0, min(4, (1 << depth) - 1) + 1))))
        free = [i for i in ([rng.randrange(1 << depth) for _ in range(8)] + list(range(4))) if i not in flagged and i < 1 << depth]
        rows.append(note_row(rng, depth, free[0], xc.BlocklistTree(depth, flagged)))
    return rows


def random_rows(rng, batch, depth):
    """Rows of uniformly random inputs (keys anywhere in u64): the witness map is defined for them too."""
    return [row(rng.randrange(R), rng.randrange(R), rng.randrange(R), [rng.randrange(R) for _ in range(depth)], rng.randrange(1 << 32),
                rng.choice([rng.randrange(1 << 64), rng.randrange(1 << 34)]), rng.choice([rng.randrange(1 << 64), rng.randrange(1 << 34)]),
                [rng.randrange(R) for _ in range(depth)], rng.randrange(1 << 32)) for _ in range(batch)]


def pack(rows):
    """The nine input buffers of og_exclusion_witness / og_groth16_prove_exclusion."""
    f = cport.frs
    return (f([r["nullifier"] for r in rows]), f([r["secret"] for r in rows]), f([r["recipient"] for r in rows]),
            f([x for r in rows for x in r["sibs"]]), [r["bits"] for r in rows], [r["low"] for r in rows], [r["next"] for r in rows],
            f([x for r in rows for x in r["xsibs"]]), [r["xbits"] for r in rows])


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


def packed_row(depth, block):
    """Index of the packed row (sum 2^k bit_k - value) * ONE = 0 of range block LOW, NEXT, GAP_LO or GAP_HI."""
    return 4 + 3 * P + depth * (2 * P + 3) + 34 * block + 33


# ---- CPU: the spec -------------------------------------------------------------------------------------------------------
def test_exclusion_sizes():
    for depth in (1, 2, 32):
        L = xc.Layout(depth)
        assert (L.n_vars, L.n_constraints) == (1964 + 1464 * depth, 1962 + 1462 * depth)
    expect = {32: (48812, 48746, 16), 2: (4892, 4886, 13), 1: (3428, 3424, 12)}
    for depth, (nv, nc, log_m) in expect.items():
        cs = xc.build_r1cs(depth)
        assert (cs.n_vars, cs.n_constraints, cs.n_pub) == (nv, nc, 4), depth
        assert g16.domain_log(cs.n_constraints, cs.n_pub) == log_m, depth
        assert ob.exclusion_r1cs_info(depth) == dict(n_constraints=nc, n_vars=nv, n_pub=4, log_m=log_m), depth
    for bad in (0, 33):
        with pytest.raises(ob.OwshenB200Error):
            ob.exclusion_r1cs_info(bad)


def test_statement_shapes_are_distinct():
    """The prover recognises a key by (n_pub, n_vars, n_constraints): no two (statement, depth) pairs share one."""
    seen = {}
    for stmt in ("withdraw", "transfer", "association", "exclusion"):
        for d in range(1, 33):
            i = api._statement_r1cs_info(stmt, d)
            shape = (i["n_pub"], i["n_vars"], i["n_constraints"])
            assert shape not in seen, (stmt, d, seen.get(shape))
            seen[shape] = (stmt, d)
    i = ob.deposit_r1cs_info()
    assert (i["n_pub"], i["n_vars"], i["n_constraints"]) not in seen


def test_blocklist_tree_spec():
    t = xc.BlocklistTree(2, [])
    assert t.keys == [0, 2 ** 32 + 1] and t.root() != mimc7.MerkleTree(2).root()       # one leaf, H(0, 2^32 + 1)
    empty = mimc7.MerkleTree(2)
    empty.insert(mimc7.hash2(0, 2 ** 32 + 1))
    assert t.root() == empty.root()
    t = xc.BlocklistTree(3, [5, 1, 5, 6])
    assert t.keys == [0, 2, 6, 7, 2 ** 32 + 1] and xc.leaves([1, 5, 6]) == [mimc7.hash2(a, b) for a, b in zip(t.keys, t.keys[1:])]
    assert [t.bracket(i) for i in (0, 2, 3, 4, 7)] == [0, 1, 1, 1, 3]
    for i in (1, 5, 6):
        with pytest.raises(ValueError):
            t.bracket(i)


@pytest.fixture(scope="module")
def cs2():
    return xc.build_r1cs(2)


def test_exclusion_witnesses_satisfy(cs2):
    rng = random.Random(1)
    for depth, cs in ((2, cs2), (3, xc.build_r1cs(3))):
        for r in edge_rows(rng, depth) + valid_rows(rng, 3, depth):
            w = spec_witness(r)
            assert cs.is_satisfied(w), r["bits"]
            assert w[xc.V_NHASH] == mimc7.multi_hash([r["nullifier"]], key=1)
            ww = wc.witness(r["nullifier"], r["secret"], r["recipient"], r["sibs"], bit_list(r["bits"], depth))
            assert w[1:4] == ww[1:4]
    # the full depth-2 tree: 2^2 - 1 flagged indices leave one note that can prove
    full = xc.BlocklistTree(2, [0, 1, 3])
    w = spec_witness(note_row(rng, 2, 2, full))
    assert cs2.is_satisfied(w) and w[xc.V_XROOT] == full.root()


def test_exclusion_mutations_are_unsatisfied(cs2):
    rng = random.Random(3)
    L = xc.Layout(2)
    bl = xc.BlocklistTree(2, [1, 2])                          # keys 0, 2, 3, 2^32 + 1
    root = bl.root()

    def claims(r):
        """The witness of row r with the published exclusion root: its failing rows."""
        w = spec_witness(r)
        w[xc.V_XROOT] = root
        return failing(cs2, w)

    good = note_row(rng, 2, 3, bl)
    assert claims(good) == []
    # a flagged index (1: x = 2 = k_1) with either bracketing leaf: leaf 0 = (0, 2) fails gap_hi, leaf 1 = (2, 3) gap_lo
    assert claims(note_row(rng, 2, 1, bl, leaf=0)) == [packed_row(2, xc.GAP_HI)]
    assert claims(note_row(rng, 2, 1, bl, leaf=1)) == [packed_row(2, xc.GAP_LO)]
    assert claims(note_row(rng, 2, 2, bl, leaf=1)) == [packed_row(2, xc.GAP_HI)]
    # a published leaf that does not bracket x
    assert claims(note_row(rng, 2, 3, bl, leaf=0)) == [packed_row(2, xc.GAP_HI)]
    assert claims(note_row(rng, 2, 0, bl, leaf=2)) == [packed_row(2, xc.GAP_LO)]
    # low and next swapped: the leaf is not the published one, and the gaps fail
    r = dict(good, low=good["next"], next=good["low"])
    bad = claims(r)
    assert cs2.n_constraints - 1 in bad and packed_row(2, xc.GAP_LO) in bad
    # low >= 2^33 in a tree that publishes it (a malicious provider): its 33 bits do not pack back to low
    for big in (2 ** 33, 2 ** 33 + 3, 2 ** 64 - 1):
        t = mimc7.MerkleTree(2)
        t.insert(mimc7.hash2(big, 2 ** 32 + 1))
        sibs, bits = t.path(0)
        r = dict(good, low=big, next=2 ** 32 + 1, xsibs=sibs, xbits=bit_word(bits))
        w = spec_witness(r)
        assert w[xc.V_XROOT] == t.root()
        assert packed_row(2, xc.LOW) in failing(cs2, w), big
    # next >= 2^33
    t = mimc7.MerkleTree(2)
    t.insert(mimc7.hash2(0, 2 ** 33 + 7))
    sibs, bits = t.path(0)
    assert packed_row(2, xc.NEXT) in failing(cs2, spec_witness(dict(good, low=0, next=2 ** 33 + 7, xsibs=sibs, xbits=bit_word(bits))))
    # one gap bit flipped: only the packed row fails
    w0 = spec_witness(good)
    for block in (xc.GAP_LO, xc.GAP_HI, xc.LOW, xc.NEXT):
        w = list(w0)
        w[L.bits(block) + 4] ^= 1
        assert failing(cs2, w) == [packed_row(2, block)], block
    # an exclusion path bit flipped
    w = list(w0)
    lv = L.level(xc.EXCL, 1)
    w[lv["bit"]] ^= 1
    assert failing(cs2, w)
    # the zero leaf: an empty position's path does not reach the published root from any (low, next)
    sibs, bits = bl.tree.path(3)
    assert claims(dict(good, xsibs=sibs, xbits=bit_word(bits))) == [cs2.n_constraints - 1]
    assert cs2.n_constraints - 1 in claims(dict(good, low=0, next=0, xsibs=sibs, xbits=bit_word(bits)))
    # a pool sibling changed while the published pool root is claimed
    w = spec_witness(good)
    w[L.level(xc.POOL, 0)["sib"]] = (w[L.level(xc.POOL, 0)["sib"]] + 1) % R
    assert failing(cs2, w)


def test_exclusion_r1cs_export_matches_spec():
    for depth in (1, 2, 32):
        cs = xc.build_r1cs(depth)
        for m in "ABC":
            assert ob.exclusion_r1cs_export(depth, m) == cs.csr(m), (depth, m)


def test_transfer_and_association_exports_unchanged_by_the_range_gadget():
    for depth in (1, 2, 32):
        for mod, export in ((tc, ob.transfer_r1cs_export), (ac, ob.association_r1cs_export)):
            cs = mod.build_r1cs(depth)
            for m in "ABC":
                assert export(depth, m) == cs.csr(m), (mod.__name__, depth, m)


def golden_row(g):
    return row(int(g["nullifier"]), int(g["secret"]), int(g["recipient"]), [int(x) for x in g["siblings"]], g["path_bits"],
               g["excl_low"], g["excl_next"], [int(x) for x in g["excl_siblings"]], g["excl_path_bits"])


def test_exclusion_golden_proof_reproduced_by_c_port():
    g = GOLD
    cs = xc.build_r1cs(g["depth"])
    pkb, vkb = cport.setup_bytes(cs, *[int(x) for x in g["toxic"]])
    assert hashlib.sha256(pkb["a"] + pkb["b1"] + pkb["b2"] + pkb["l"] + pkb["h"]).hexdigest() == g["pk_queries_sha256"]
    v = g["vk"]
    assert (vkb["alpha1"] + vkb["beta2"] + vkb["gamma2"] + vkb["delta2"] + vkb["ic"]).hex() == v["alpha1"] + v["beta2"] + v["gamma2"] + v["delta2"] + v["ic"]
    w = spec_witness(golden_row(g))
    assert cs.is_satisfied(w)
    assert w[xc.V_XROOT] == xc.BlocklistTree(g["depth"], g["flagged"]).root()
    wit = cport.frs(w)
    assert hashlib.sha256(wit).hexdigest() == g["witness_sha256"]
    assert cport.unfr(wit[32:32 * 5]) == [int(x) for x in g["public"]]
    assert cport.Prover(cs, pkb).prove(wit, int(g["r"]), int(g["s"])).hex() == g["proof"]
    assert ob.verify(vk_blob(vkb, 4), wit[32:32 * 5], bytes.fromhex(g["proof"]))


def test_exclusion_set_validates_before_any_gpu_work():
    for depth, flagged in ((0, []), (33, []), (2, [4]), (2, [-1]), (2, [0, 1, 2, 3]), (1, [0, 1])):
        with pytest.raises(ValueError):
            ob.ExclusionSet(None, depth, flagged)


# ---- GPU -----------------------------------------------------------------------------------------------------------------
_KEYS = {}


def exclusion_keys(ctx, depth):
    """(pk, vk, r1cs, oracle pk bytes, oracle vk bytes) of the depth-`depth` exclusion statement, made once per process."""
    if depth not in _KEYS:
        rng = random.Random(70 + depth)
        tw = [rng.randrange(1, R) for _ in range(5)]
        pk, vk = ob.setup_exclusion(ctx, depth, *tw)
        cs = xc.build_r1cs(depth)
        pkb, vkb = cport.setup_bytes(cs, *tw)
        _KEYS[depth] = (pk, vk, cs, pkb, vkb)
    return _KEYS[depth]


def proofs_verify(vk, proofs, pub, batch):
    return [ob.verify(vk, pub[128 * i:128 * i + 128], proofs[256 * i:256 * i + 256]) for i in range(batch)]


@pytest.mark.gpu
def test_exclusion_witness_matches_oracle(ctx):
    rng = random.Random(71)
    # depth 2: 40 rows with every edge row, the soundness mutations' rows and random keys anywhere in u64
    bl = xc.BlocklistTree(2, [1, 2])
    mutated = [note_row(rng, 2, 1, bl, leaf=0), note_row(rng, 2, 1, bl, leaf=1), note_row(rng, 2, 3, bl, leaf=0),
               note_row(rng, 2, 0, bl, leaf=2)]
    swapped = dict(mutated[0], low=mutated[0]["next"], next=mutated[0]["low"])
    wide = [dict(mutated[1], low=lo, next=nx) for lo, nx in ((2 ** 33, 2 ** 32 + 1), (2 ** 64 - 1, 0), (0, 2 ** 64 - 1), (2 ** 64 - 1, 2 ** 64 - 1))]
    rows = edge_rows(rng, 2) + mutated + [swapped] + wide
    rows += valid_rows(rng, 6, 2)
    rows += random_rows(rng, 40 - len(rows), 2)
    assert len(rows) == 40
    assert ctx.exclusion_witness(2, *pack(rows)) == oracle_witnesses(rows)
    rows = edge_rows(rng, 32)[:4] + random_rows(rng, 2, 32)
    assert ctx.exclusion_witness(32, *pack(rows)) == oracle_witnesses(rows)
    # a field input >= r in any of the five field arrays
    rows = valid_rows(rng, 2, 2)
    for k in (0, 1, 2, 3, 7):
        p = list(pack(rows))
        p[k] = R.to_bytes(32, "little") + p[k][32:]
        with pytest.raises(ob.OwshenB200Error) as e:
            ctx.exclusion_witness(2, *p)
        assert e.value.code == -4 or "encoding" in str(e.value).lower(), k
    # wrong lengths
    p = pack(rows)
    for k, bad in ((3, p[3][:-32]), (4, p[4][:1]), (5, p[5] + [0]), (6, p[6][:1]), (7, p[7] + bytes(32)), (8, p[8] + [0])):
        q = list(p)
        q[k] = bad
        with pytest.raises(ValueError):
            ctx.exclusion_witness(2, *q)


@pytest.mark.gpu
def test_setup_exclusion_matches_oracle(ctx):
    for depth in (2, 32):
        pk, vk, cs, pkb, vkb = exclusion_keys(ctx, depth)
        assert pk == pk_blob(cs, pkb, 0), depth
        assert vk == vk_blob(vkb, 4), depth


@pytest.mark.gpu
def test_exclusion_key_from_ceremony(ctx):
    """One phase-1 contribution (t, a, b), then the depth-2 key: before phase 2, gamma = delta = 1 (DESIGN.md section 4b)."""
    rng = random.Random(72)
    t, a, b = (rng.randrange(1, R) for _ in range(3))
    acc0 = ob.ptau_new(ctx, 13)                           # the depth-2 exclusion domain is 2^13
    acc1, rec = ob.ptau_contribute(ctx, acc0, [t, a, b], [rng.randrange(1, R) for _ in range(3)])
    assert ob.ptau_verify(ctx, acc0, acc1, rec)
    pk, vk = ob.ptau_prepare_exclusion(ctx, acc1, 2)
    assert (pk, vk) == ob.setup_exclusion(ctx, 2, t, a, b, 1, 1)
    cs = xc.build_r1cs(2)
    pkb, vkb = cport.setup_bytes(cs, t, a, b, 1, 1)
    assert pk == pk_blob(cs, pkb, 0) and vk == vk_blob(vkb, 4)
    PK = ob.ProvingKey(ctx, pk)
    try:
        assert (PK.exclusion_depth, PK.association_depth) == (2, None)
    finally:
        PK.close()


@pytest.mark.gpu
@pytest.mark.parametrize("depth,batch", [(2, 40), (32, 3)])
def test_prove_exclusion_matches_oracle(ctx, monkeypatch, depth, batch):
    pk, vk, cs, pkb, vkb = exclusion_keys(ctx, depth)
    rng = random.Random(73 + depth)
    rows = (edge_rows(rng, depth) + valid_rows(rng, batch, depth))[:batch]
    rs = cport.frs([rng.randrange(R) for _ in range(2 * batch)])
    wit = oracle_witnesses(rows)
    exp = cport.Prover(cs, pkb).prove_batch(wit, rs)
    results = []
    for env in (dict(), dict(OG_CHUNK=3, OG_LANES=2)):
        set_env(monkeypatch, **env)
        PK = ob.ProvingKey(ctx, pk)
        try:
            assert (PK.n_vars, PK.n_pub, PK.depth, PK.exclusion_depth, PK.association_depth) == (cs.n_vars, 4, 0, depth, None)
            results.append(PK.prove_exclusion(*pack(rows), rs))
        finally:
            PK.close()
    set_env(monkeypatch)
    nv = cs.n_vars
    for proofs, pub in results:
        assert proofs == exp
        assert pub == b"".join(wit[32 * nv * i + 32:32 * nv * i + 32 * 5] for i in range(batch))
    proofs, pub = results[0]
    assert all(proofs_verify(vk, proofs, pub, batch))
    bad = bytearray(pub[:128]); bad[96] ^= 1          # another exclusion root
    assert not ob.verify(vk, bytes(bad), proofs[:256])


@pytest.mark.gpu
def test_prove_exclusion_dev_matches_host_entry_point(ctx):
    import torch
    pk = exclusion_keys(ctx, 2)[0]
    rng = random.Random(74)
    batch = 5
    rows = valid_rows(rng, batch, 2)
    rs = cport.frs([rng.randrange(R) for _ in range(2 * batch)])
    p = pack(rows)
    PK = ob.ProvingKey(ctx, pk)
    try:
        proofs, pub = PK.prove_exclusion(*p, rs)
        words = lambda xs: struct.pack(f"<{len(xs)}I", *xs)
        u64 = lambda xs: struct.pack(f"<{len(xs)}Q", *xs)
        dev = lambda b: torch.frombuffer(bytearray(b), dtype=torch.uint8).to("cuda")
        d_in = [dev(x) for x in (p[0], p[1], p[2], p[3], words(p[4]), u64(p[5]), u64(p[6]), p[7], words(p[8]), rs)]
        d_pr = torch.zeros(256 * batch, dtype=torch.uint8, device="cuda")
        d_pub = torch.zeros(128 * batch, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        rc = api.lib().og_groth16_prove_exclusion_dev(ctx._h, PK._h, *[api._ptr(t) for t in d_in[:9]], batch, api._ptr(d_in[9]),
                                                      api._ptr(d_pr), api._ptr(d_pub))
        assert rc == 0
        ctx.sync()
        assert bytes(d_pr.cpu().numpy()) == proofs and bytes(d_pub.cpu().numpy()) == pub
    finally:
        PK.close()


@pytest.mark.gpu
def test_exclusion_golden_proof(ctx):
    g = GOLD
    pk, vk = ob.setup_exclusion(ctx, g["depth"], *[int(x) for x in g["toxic"]])
    v = g["vk"]
    assert vk[12:].hex() == v["alpha1"] + v["beta2"] + v["gamma2"] + v["delta2"] + v["ic"]
    rs = bn.fr_to_bytes(int(g["r"])) + bn.fr_to_bytes(int(g["s"]))
    PK = ob.ProvingKey(ctx, pk)
    try:
        proofs, pub = PK.prove_exclusion(*pack([golden_row(g)]), rs)
    finally:
        PK.close()
    assert proofs.hex() == g["proof"]
    assert cport.unfr(pub) == [int(x) for x in g["public"]]
    assert ob.verify(vk, pub, proofs)


@pytest.mark.gpu
def test_flagged_note_fails_alone(ctx):
    """A flagged note forced into a batch with a published leaf that does not bracket it is proved like any other; checked
    against the published roots, its proof fails and the rest of the batch verifies."""
    pk, vk = exclusion_keys(ctx, 2)[:2]
    rng = random.Random(75)
    bl = xc.BlocklistTree(2, [1])
    rows = [note_row(rng, 2, rng.choice([0, 2, 3]), bl) for _ in range(8)]
    rows[3] = note_row(rng, 2, 1, bl, leaf=rng.choice([0, 1]))
    rs = cport.frs([rng.randrange(R) for _ in range(16)])
    PK = ob.ProvingKey(ctx, pk)
    try:
        proofs, pub = PK.prove_exclusion(*pack(rows), rs)
    finally:
        PK.close()
    ok = []
    for i in range(8):
        p = cport.unfr(pub[128 * i:128 * i + 128])
        assert p[3] == bl.root(), i          # the path is a published one: only the range checks fail
        ok.append(ob.verify(vk, cport.frs(p[:3] + [bl.root()]), proofs[256 * i:256 * i + 256]))
    assert ok == [i != 3 for i in range(8)]


# every statement's prover: (name, number of input arrays)
_PROVERS = (("withdraw", 5), ("deposit", 3), ("transfer", 11), ("association", 7), ("exclusion", 9))


@pytest.mark.gpu
def test_every_prover_refuses_the_other_statements_keys(ctx):
    import torch
    d_buf = torch.zeros(1 << 16, dtype=torch.uint8, device="cuda")
    d = api._ptr(d_buf)                                   # every device argument of the _dev entry points
    h = bytes(1 << 16)                                    # every host input of the host entry points
    rng = random.Random(76)
    tw = [rng.randrange(1, R) for _ in range(5)]
    keys = {"withdraw": ob.setup_withdraw(ctx, 2, *tw)[0], "deposit": ob.setup_deposit(ctx, *tw)[0],
            "transfer": ob.setup_transfer(ctx, 2, *tw)[0], "association": ob.setup_association(ctx, 2, *tw)[0],
            "exclusion": exclusion_keys(ctx, 2)[0]}
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
        finally:
            PK.close()
    PK = ob.ProvingKey(ctx, keys["exclusion"])
    try:
        rows = valid_rows(rng, 2, 2)
        assert len(PK.prove_exclusion(*pack(rows), cport.frs([rng.randrange(R) for _ in range(4)]))[0]) == 512   # still usable
    finally:
        PK.close()


@pytest.mark.gpu
def test_exclusion_set_matches_oracle_tree(ctx):
    rng = random.Random(77)
    for depth, flagged in ((1, []), (1, [1]), (2, [0, 1, 2]), (3, [6, 2, 2, 4]), (5, rng.sample(range(32), 9)), (8, [])):
        xs = ob.ExclusionSet(ctx, depth, flagged)
        spec = xc.BlocklistTree(depth, flagged)
        assert int.from_bytes(xs.root(), "little") == spec.root(), (depth, flagged)
        assert len(xs) == len(spec.flagged) and xs.keys == spec.keys
        assert all((i in xs) == (i in spec.flagged) for i in range(1 << depth))
        free = [i for i in range(1 << depth) if i not in spec.flagged]
        low, nxt, sibs, bits = xs.witness(free)
        for k, i in enumerate(free):
            s_low, s_next, s_sibs, s_bits = spec.witness(i)
            assert (low[k], nxt[k], cport.unfr(sibs[32 * depth * k:32 * depth * (k + 1)]), bits[k]) == (s_low, s_next, s_sibs, bit_word(s_bits))
        for i in spec.flagged:
            with pytest.raises(ValueError, match=str(i)):
                xs.witness([free[0], i])
    # 2^16 flagged indices at depth 20: sampled paths reach the root through og_mimc7_merkle_paths
    depth = 20
    flagged = rng.sample(range(1 << depth), 1 << 16)
    xs = ob.ExclusionSet(ctx, depth, flagged)
    assert len(xs) == 1 << 16
    fs = set(flagged)
    notes = [i for i in (rng.randrange(1 << depth) for _ in range(64)) if i not in fs][:32]
    low, nxt, sibs, bits = xs.witness(notes)
    assert all(lo < i + 1 < nx for lo, i, nx in zip(low, notes, nxt))
    leaves = cport.frs([mimc7.hash2(lo, nx) for lo, nx in zip(low, nxt)])
    nodes = ctx.merkle_paths(leaves, sibs, bits, depth)
    stride = 32 * (depth + 1)
    assert all(nodes[stride * k + 32 * depth:stride * (k + 1)] == xs.root() for k in range(len(notes)))


@pytest.mark.gpu
def test_deposit_to_exclusion_withdraw_chain(ctx):
    """Deposits' commitments in a depth-32 pool tree (GPU MerkleTree) and a provider's ExclusionSet over some of their
    indices; depth-32 exclusion withdrawals of the unflagged notes verify against both published roots, and ExclusionSet
    refuses to give a flagged note a witness."""
    rng = random.Random(78)
    n = 6
    notes = [(rng.randrange(R), rng.randrange(R)) for _ in range(n)]
    cms = [mimc7.multi_hash(list(x)) for x in notes]
    pool = ob.MerkleTree(ctx, 32)
    pool.insert_batch([rng.randrange(R) for _ in range(3)])
    pool_idx = pool.insert_batch(cms)
    flagged_notes = [1, 4]
    xs = ob.ExclusionSet(ctx, 32, [pool_idx[k] for k in flagged_notes] + [0, 1 << 20])
    as_int = lambda b: int.from_bytes(b, "little")
    roots = (as_int(pool.root()), as_int(xs.root()))
    for k in flagged_notes:
        with pytest.raises(ValueError, match=str(pool_idx[k])):
            xs.witness([pool_idx[k]])
    spenders = [k for k in range(n) if k not in flagged_notes]
    sibs, bits = pool.paths([pool_idx[k] for k in spenders])
    low, nxt, xsibs, xbits = xs.witness([pool_idx[k] for k in spenders])
    recipients = [rng.randrange(1 << 160) for _ in spenders]
    pk, vk = exclusion_keys(ctx, 32)[:2]
    PK = ob.ProvingKey(ctx, pk)
    try:
        proofs, pub = PK.prove_exclusion(cport.frs([notes[k][0] for k in spenders]), cport.frs([notes[k][1] for k in spenders]),
                                         cport.frs(recipients), sibs, bits, low, nxt, xsibs, xbits,
                                         cport.frs([rng.randrange(R) for _ in range(2 * len(spenders))]))
    finally:
        PK.close()
    for i, k in enumerate(spenders):
        p = cport.unfr(pub[128 * i:128 * i + 128])
        assert p == [roots[0], mimc7.multi_hash([notes[k][0]], key=1), recipients[i], roots[1]], k
        assert ob.verify(vk, cport.frs(p), proofs[256 * i:256 * i + 256]), k


@pytest.mark.gpu
def test_exclusion_prover_plan_and_batch_above_default_chunk(monkeypatch):
    """The depth-32 key's default chunk is what the 28 GiB lane budget gives; chunk + 1 proofs at default settings run as two
    chunks on two lanes, match the oracle and verify."""
    import torch
    set_env(monkeypatch)
    c = ob.Context(0)          # its own scratch: the session context keeps what earlier tests grew
    try:
        pk, vk, cs, pkb, vkb = exclusion_keys(c, 32)
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
            rng = random.Random(79)
            rows = random_rows(rng, batch, 32)
            for i, r in zip((0, chunk - 1, chunk), valid_rows(rng, 3, 32)):
                rows[i] = r
            rs = cport.frs([rng.randrange(R) for _ in range(2 * batch)])
            proofs, pub = PK.prove_exclusion(*pack(rows), rs)
        finally:
            PK.close()
    finally:
        c.close()
    prover = cport.Prover(cs, pkb)
    for i in (0, chunk - 1, chunk):
        wit = cport.frs(spec_witness(rows[i]))
        assert proofs[256 * i:256 * i + 256] == prover.prove_batch(wit, rs[64 * i:64 * i + 64]), i
        assert ob.verify(vk, pub[128 * i:128 * i + 128], proofs[256 * i:256 * i + 256]), i
