"""The deposit statement (oracle/deposit_circuit.py == csrc/withdraw_circuit.hpp: DepositBuilder): its spec, the library's
R1CS export, GPU witness, setup and batched prover against the oracle, deposits opened by the withdraw statement, and the
prover's window bits chosen from the key's size."""
import hashlib
import json
import os
import random

import pytest

import owshen_b200 as ob
from owshen_b200 import api
from oracle import bn254 as bn
from oracle import cport, mimc7
from oracle import deposit_circuit as dc
from oracle import groth16 as g16
from oracle import withdraw_circuit as wc
from tests.helpers import pk_blob, vk_blob, withdraw_keys32

R = bn.R
GOLD = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "deposit_vectors.json")))
EDGE = [0, 1, R - 1]


# ---- mirror of groth16.cu: pk_load's window rule ------------------------------------------------------------------------
def window_rule(n):
    """The c in [2, 16] minimising n * ceil(255 / c) + 2.3 * 2^(c-1) (compared in tenths); ties to the smaller c."""
    return min(range(2, 17), key=lambda c: (10 * n * -(-255 // c) + 23 * (1 << (c - 1)), c))


def msm_sizes(cs):
    """Points of the prover's A, B and C' MSMs for a key of this R1CS (B's support = variables with a B term)."""
    m = 1 << g16.domain_log(cs.n_constraints, cs.n_pub)
    n_supp = len({i for row in cs.B for i in row})
    return cs.n_vars + 2, n_supp + 2, cs.n_vars - cs.n_pub - 1 + n_supp + m + 1


def expected_window_bits(cs):
    return tuple(window_rule(n) for n in msm_sizes(cs))


def rand_deposits(rng, batch):
    nul = cport.frs([rng.randrange(R) for _ in range(batch)])
    sec = cport.frs([rng.randrange(R) for _ in range(batch)])
    dep = cport.frs([rng.randrange(1 << 160) for _ in range(batch)])
    return nul, sec, dep


def oracle_witnesses(nul, sec, dep):
    u = cport.unfr
    return b"".join(cport.frs(dc.witness(n, s, d)) for n, s, d in zip(u(nul), u(sec), u(dep)))


# ---- CPU -----------------------------------------------------------------------------------------------------------------
def test_deposit_witness_satisfies_r1cs():
    cs = dc.build_r1cs()
    L = dc.Layout()
    assert (cs.n_vars, cs.n_constraints, cs.n_pub) == (735, 731, 2) == (L.n_vars, L.n_constraints, dc.N_PUB)
    assert g16.domain_log(cs.n_constraints, cs.n_pub) == 10
    rng = random.Random(1)
    for n, s, d in [(rng.randrange(R), rng.randrange(R), rng.randrange(R)), (0, 0, 0), (1, R - 1, 0), (R - 1, 1, R - 1)]:
        w = dc.witness(n, s, d)
        assert cs.is_satisfied(w)
        bad = list(w); bad[1] = (bad[1] + 1) % R
        assert not cs.is_satisfied(bad)


def test_deposit_commitment_is_a_withdraw_leaf():
    rng = random.Random(2)
    for n, s in [(rng.randrange(R), rng.randrange(R)), (0, 0), (R - 1, 1)]:
        w = dc.witness(n, s, rng.randrange(R))
        assert w[1] == mimc7.multi_hash([n, s])
        ww = wc.witness(n, s, 5, [rng.randrange(R)], [1])
        assert w[1] == ww[wc.Layout(1).cm_out]
        # the commitment block is laid out and filled exactly like the withdraw statement's
        assert w[dc.Layout().cm_base:] == ww[wc.Layout(1).cm_base:wc.Layout(1).cm_out + 1]


def test_deposit_r1cs_export_matches_spec():
    cs = dc.build_r1cs()
    info = ob.deposit_r1cs_info()
    assert info == dict(n_constraints=cs.n_constraints, n_vars=cs.n_vars, n_pub=cs.n_pub, log_m=10)
    for m in "ABC":
        assert ob.deposit_r1cs_export(m) == cs.csr(m), m


def test_deposit_golden_proof_reproduced_by_c_port():
    g = GOLD
    cs = dc.build_r1cs()
    pkb, vkb = cport.setup_bytes(cs, *[int(x) for x in g["toxic"]])
    assert hashlib.sha256(pkb["a"] + pkb["b1"] + pkb["b2"] + pkb["l"] + pkb["h"]).hexdigest() == g["pk_queries_sha256"]
    v = g["vk"]
    assert (vkb["alpha1"] + vkb["beta2"] + vkb["gamma2"] + vkb["delta2"] + vkb["ic"]).hex() == v["alpha1"] + v["beta2"] + v["gamma2"] + v["delta2"] + v["ic"]
    wit = cport.frs(dc.witness(int(g["nullifier"]), int(g["secret"]), int(g["depositor"])))
    assert hashlib.sha256(wit).hexdigest() == g["witness_sha256"]
    assert cport.unfr(wit[32:96]) == [int(x) for x in g["public"]]
    assert cport.Prover(cs, pkb).prove(wit, int(g["r"]), int(g["s"])).hex() == g["proof"]
    assert ob.verify(vk_blob(vkb, 2), wit[32:96], bytes.fromhex(g["proof"]))


def test_window_rule_keeps_the_depth32_withdraw_windows():
    """The rule reproduces the measured optimum of the depth-32 withdraw key, and gives the deposit key smaller windows."""
    cs = wc.build_r1cs(32)
    assert msm_sizes(cs) == (24526, 12294, 69581)
    assert expected_window_bits(cs) == (15, 15, 16)
    assert expected_window_bits(dc.build_r1cs()) == (11, 10, 12)
    assert window_rule(0) == 2 and window_rule(1 << 30) == 16


# ---- GPU -----------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def deposit_keys(ctx):
    rng = random.Random(30)
    tw = [rng.randrange(1, R) for _ in range(5)]
    pk, vk = ob.setup_deposit(ctx, *tw)
    cs = dc.build_r1cs()
    pkb, vkb = cport.setup_bytes(cs, *tw)
    return pk, vk, cs, pkb, vkb


def set_env(monkeypatch, **env):
    for k in ("OG_CHUNK", "OG_LANES", "OG_C_A", "OG_C_B", "OG_C_C", "OG_WINDOW_BITS"):
        if env.get(k) is None:
            monkeypatch.delenv(k, raising=False)
        else:
            monkeypatch.setenv(k, str(env[k]))


@pytest.mark.gpu
def test_deposit_witness_matches_oracle(ctx):
    rng = random.Random(31)
    nul, sec, dep = rand_deposits(rng, 37)
    assert ctx.deposit_witness(nul, sec, dep) == oracle_witnesses(nul, sec, dep)
    edges = [(n, s, d) for n in EDGE for s in EDGE for d in EDGE]
    nul, sec, dep = (cport.frs([e[k] for e in edges]) for k in range(3))
    assert ctx.deposit_witness(nul, sec, dep) == oracle_witnesses(nul, sec, dep)
    with pytest.raises(ob.OwshenB200Error):
        ctx.deposit_witness(R.to_bytes(32, "little"), sec[:32], dep[:32])


@pytest.mark.gpu
def test_setup_deposit_matches_oracle(ctx, deposit_keys):
    pk, vk, cs, pkb, vkb = deposit_keys
    assert pk == pk_blob(cs, pkb, 0)
    assert vk == vk_blob(vkb, 2)


@pytest.mark.gpu
def test_prove_deposit_matches_oracle_in_chunks_and_lanes(ctx, deposit_keys, monkeypatch):
    pk, vk, cs, pkb, vkb = deposit_keys
    rng = random.Random(32)
    batch = 257
    nul, sec, dep = rand_deposits(rng, batch)
    rs = cport.frs([rng.randrange(R) for _ in range(2 * batch)])
    wit = oracle_witnesses(nul, sec, dep)
    exp = cport.Prover(cs, pkb).prove_batch(wit, rs)
    nv = cs.n_vars
    results = []
    for lanes in (1, 2):
        set_env(monkeypatch, OG_CHUNK=100, OG_LANES=lanes)
        PK = ob.ProvingKey(ctx, pk)
        try:
            assert (PK.n_vars, PK.n_pub, PK.log_m, PK.depth) == (735, 2, 10, 0)
            results.append(PK.prove_deposit(nul, sec, dep, rs))
            assert PK.prove_deposit(nul, sec, dep, rs, want_public=False) == (results[-1][0], None)
        finally:
            PK.close()
    set_env(monkeypatch)
    (proofs, pub), (proofs2, pub2) = results
    assert proofs == exp and proofs2 == exp and pub2 == pub
    for i in range(batch):
        x = pub[64 * i:64 * i + 64]
        assert x == wit[32 * nv * i + 32:32 * nv * i + 96], i
        assert cport.unfr(x) == [mimc7.multi_hash(cport.unfr(nul[32 * i:32 * i + 32] + sec[32 * i:32 * i + 32])), cport.unfr(dep[32 * i:32 * i + 32])[0]]
        assert ob.verify(vk, x, proofs[256 * i:256 * i + 256]), i
    for i in (0, 99, 100, 256):
        for byte in (0, 40):
            bad = bytearray(pub[64 * i:64 * i + 64]); bad[byte] ^= 1
            assert not ob.verify(vk, bytes(bad), proofs[256 * i:256 * i + 256]), (i, byte)


@pytest.mark.gpu
def test_prove_deposit_dev_matches_host_entry_point(ctx, deposit_keys):
    import torch
    pk = deposit_keys[0]
    rng = random.Random(33)
    batch = 5
    nul, sec, dep = rand_deposits(rng, batch)
    rs = cport.frs([rng.randrange(R) for _ in range(2 * batch)])
    PK = ob.ProvingKey(ctx, pk)
    try:
        proofs, pub = PK.prove_deposit(nul, sec, dep, rs)
        dev = lambda b: torch.frombuffer(bytearray(b), dtype=torch.uint8).to("cuda")
        d_in = [dev(x) for x in (nul, sec, dep, rs)]
        d_pr = torch.zeros(256 * batch, dtype=torch.uint8, device="cuda")
        d_pub = torch.zeros(64 * batch, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        rc = api.lib().og_groth16_prove_deposit_dev(ctx._h, PK._h, *[api._ptr(t) for t in d_in[:3]], batch, api._ptr(d_in[3]),
                                                    api._ptr(d_pr), api._ptr(d_pub))
        assert rc == 0
        ctx.sync()
        assert bytes(d_pr.cpu().numpy()) == proofs and bytes(d_pub.cpu().numpy()) == pub
    finally:
        PK.close()


@pytest.mark.gpu
def test_deposit_golden_proof(ctx):
    g = GOLD
    pk, vk = ob.setup_deposit(ctx, *[int(x) for x in g["toxic"]])
    v = g["vk"]
    assert vk[12:].hex() == v["alpha1"] + v["beta2"] + v["gamma2"] + v["delta2"] + v["ic"]
    f = lambda k: bn.fr_to_bytes(int(g[k]))
    PK = ob.ProvingKey(ctx, pk)
    try:
        proofs, pub = PK.prove_deposit(f("nullifier"), f("secret"), f("depositor"), f("r") + f("s"))
    finally:
        PK.close()
    assert proofs.hex() == g["proof"]
    assert cport.unfr(pub) == [int(x) for x in g["public"]]
    assert ob.verify(vk, pub, proofs)
    wit = ctx.deposit_witness(f("nullifier"), f("secret"), f("depositor"))
    assert hashlib.sha256(wit).hexdigest() == g["witness_sha256"]


@pytest.mark.gpu
def test_deposit_then_withdraw(ctx, deposit_keys):
    """Deposits proved, their commitments inserted into a depth-32 tree, and the same notes withdrawn against its root."""
    pk_d, vk_d = deposit_keys[:2]
    pk_w, vk_w = withdraw_keys32(ctx)[:2]
    rng = random.Random(34)
    batch = 6
    nul, sec, dep = rand_deposits(rng, batch)
    rs = cport.frs([rng.randrange(R) for _ in range(2 * batch)])
    PK = ob.ProvingKey(ctx, pk_d)
    try:
        proofs, pub = PK.prove_deposit(nul, sec, dep, rs)
    finally:
        PK.close()
    commitments = [pub[64 * i:64 * i + 32] for i in range(batch)]
    assert all(ob.verify(vk_d, pub[64 * i:64 * i + 64], proofs[256 * i:256 * i + 256]) for i in range(batch))
    tree = ob.MerkleTree(ctx, 32)
    tree.insert_batch([rng.randrange(R) for _ in range(3)])       # other notes before and between the deposits
    idx = tree.insert_batch(commitments[:4])
    tree.insert(rng.randrange(R))
    idx += tree.insert_batch(commitments[4:])
    sib, bits = tree.paths(idx)
    rec = cport.frs([rng.randrange(1 << 160) for _ in range(batch)])
    rs_w = cport.frs([rng.randrange(R) for _ in range(2 * batch)])
    PK = ob.ProvingKey(ctx, pk_w)
    try:
        wproofs, wpub = ob.prove(PK, nul, sec, rec, sib, bits, rs_w)
    finally:
        PK.close()
    for i in range(batch):
        x = wpub[96 * i:96 * i + 96]
        assert x[:32] == tree.root(), i
        assert cport.unfr(x[32:64]) == [mimc7.multi_hash(cport.unfr(nul[32 * i:32 * i + 32]), key=1)], i
        assert ob.verify(vk_w, x, wproofs[256 * i:256 * i + 256]), i


def _generic_key(ctx, n_vars, n_pub, rng):
    """A key of a small R1CS that is not the deposit statement's shape."""
    cs = wc.R1CS(n_vars, n_pub)
    for j in range(n_vars - 1):
        cs.add({j: 1}, {j: 1}, {j + 1: 1})
    return ob.setup_r1cs(ctx, cs.n_vars, cs.n_pub, cs.csr("A"), cs.csr("B"), cs.csr("C"), *[rng.randrange(1, R) for _ in range(5)])[0]


@pytest.mark.gpu
def test_prove_deposit_and_withdraw_refuse_each_others_keys(ctx, deposit_keys):
    import torch
    pk_d = deposit_keys[0]
    rng = random.Random(35)
    nul, sec, dep = rand_deposits(rng, 2)
    rs = cport.frs([rng.randrange(R) for _ in range(4)])
    tw = [rng.randrange(1, R) for _ in range(5)]
    d_buf = torch.zeros(1 << 16, dtype=torch.uint8, device="cuda")
    d = api._ptr(d_buf)      # every device argument of the _dev entry points
    others = [ob.setup_withdraw(ctx, 2, *tw)[0], _generic_key(ctx, 735, 2, rng), _generic_key(ctx, 735, 1, rng)]
    for pk in others:
        PK = ob.ProvingKey(ctx, pk)
        try:
            with pytest.raises(ob.OwshenB200Error) as e:
                PK.prove_deposit(nul, sec, dep, rs)
            assert e.value.code == api.OG_E_INVALID
            for b in (2, 0):      # the key is wrong whatever the batch
                rc = api.lib().og_groth16_prove_deposit(ctx._h, PK._h, nul, sec, dep, b, rs, api.C.create_string_buffer(512), None)
                assert rc == api.OG_E_INVALID, b
                assert api.lib().og_groth16_prove_deposit_dev(ctx._h, PK._h, d, d, d, b, d, d, None) == api.OG_E_INVALID, b
        finally:
            PK.close()
    PK = ob.ProvingKey(ctx, pk_d)
    try:
        assert PK.depth == 0
        with pytest.raises(ValueError):
            ob.prove(PK, nul, sec, dep, bytes(64), [0, 0], rs)
        bits = (api.C.c_uint32 * 2)(0, 0)
        for b in (2, 0):
            rc = api.lib().og_groth16_prove_withdraw(ctx._h, PK._h, nul, sec, dep, bytes(64), bits, b, rs, api.C.create_string_buffer(512),
                                                     None)
            assert rc == api.OG_E_INVALID, b
            assert api.lib().og_groth16_prove_withdraw_dev(ctx._h, PK._h, d, d, d, d, d, b, d, d, None) == api.OG_E_INVALID, b
        assert len(PK.prove_deposit(nul, sec, dep, rs)[0]) == 512          # the context is still usable
    finally:
        PK.close()


@pytest.mark.gpu
def test_window_bits_from_key_size(ctx, deposit_keys, monkeypatch):
    pk_d, vk_d, cs_d = deposit_keys[:3]
    pk_w, cs_w = withdraw_keys32(ctx)[0], withdraw_keys32(ctx)[2]
    set_env(monkeypatch)
    for pk, cs in ((pk_w, cs_w), (pk_d, cs_d)):
        PK = ob.ProvingKey(ctx, pk)
        try:
            assert PK.window_bits == expected_window_bits(cs)
        finally:
            PK.close()
    assert expected_window_bits(cs_w) == (15, 15, 16)
    rule = expected_window_bits(cs_d)
    for env, want in ((dict(OG_C_A=9), (9, rule[1], rule[2])),
                      (dict(OG_WINDOW_BITS=13, OG_C_B=7), (13, 7, 13)),
                      (dict(OG_C_C=17, OG_C_A=1), rule),                  # out of range: the rule
                      (dict(OG_WINDOW_BITS="abc"), rule)):
        set_env(monkeypatch, **env)
        PK = ob.ProvingKey(ctx, pk_d)
        try:
            assert PK.window_bits == want, env
        finally:
            PK.close()
    set_env(monkeypatch)


@pytest.mark.gpu
def test_deposit_proofs_do_not_depend_on_window_bits(ctx, deposit_keys, monkeypatch):
    pk, vk, cs, pkb, vkb = deposit_keys
    rng = random.Random(36)
    batch = 9
    nul, sec, dep = rand_deposits(rng, batch)
    rs = cport.frs([rng.randrange(R) for _ in range(2 * batch)])
    exp = cport.Prover(cs, pkb).prove_batch(oracle_witnesses(nul, sec, dep), rs)
    for env, bits in ((dict(), expected_window_bits(cs)), (dict(OG_C_A=8, OG_C_B=9, OG_C_C=10), (8, 9, 10)),
                      (dict(OG_WINDOW_BITS=16), (16, 16, 16))):
        set_env(monkeypatch, **env)
        PK = ob.ProvingKey(ctx, pk)
        try:
            assert PK.window_bits == bits
            assert PK.prove_deposit(nul, sec, dep, rs)[0] == exp, env
        finally:
            PK.close()
    set_env(monkeypatch)
