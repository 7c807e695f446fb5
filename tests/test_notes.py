"""Encrypted note delivery (oracle/notes.py == csrc/note_core.cuh): the spec against its golden vectors and its properties,
the host-compiled core against the spec, the transfer envelope, and on the GPU the public keys, encryption and scanning
entry points against the spec, at scale, and through a deposit -> withdrawal-with-change chain."""
import ctypes as C
import json
import os
import random
import struct
import subprocess

import numpy as np
import pytest

import owshen_b200 as ob
from owshen_b200 import api, formats
from oracle import babyjubjub as bjj
from oracle import cport
from oracle import notes as N
from oracle.bn254 import R
from tests.golden.gen_note_golden import non_decompressing_x, set_word, shift_record, torsion_points

L = N.L
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = json.load(open(os.path.join(ROOT, "tests", "golden", "note_vectors.json")))
fr = lambda xs: b"".join(x.to_bytes(32, "little") for x in xs)
words = lambda b, k: [b[k * i:k * i + k] for i in range(len(b) // k)]


def rand_note(rng, amount=None):
    return (rng.randrange(R), rng.randrange(R), rng.randrange(R), rng.randrange(1 << 64) if amount is None else amount)


def golden_encryptions():
    e = GOLD["encryptions"]
    pks = [(int(x["pk_x"]), x["pk_odd"]) for x in e]
    notes = [tuple(int(v) for v in x["note"]) for x in e]
    return pks, notes, [int(x["e"]) for x in e], e


def golden_scan():
    s = GOLD["scan"]
    return ([bytes.fromhex(r) for r in s["records"]], [int(c) for c in s["commitments"]], s["owners"],
            [bytes.fromhex(p) for p in s["plaintexts"]])


def mixed_records(rng, keys, n):
    """n records mixing notes owned by each key, foreign notes, tampered words, torsion-shifted points and every malformed
    kind, with their commitments (spec encryption)."""
    torsion = torsion_points()
    bad_x = non_decompressing_x()
    recs, cms = [], []
    for i in range(n):
        kind = i % 8
        owner_key = keys[i % len(keys)] if kind != 1 else rng.randrange(1, R)
        st, rec, cm = N.encrypt(N.public_key(owner_key), rand_note(rng, [0, (1 << 64) - 1, None][i % 3]), rng.randrange(1, R))
        assert st == N.ENC_OK
        if kind == 2:                                  # a tampered word: not owned (or malformed when it leaves the field)
            k = rng.randrange(5)
            w = int.from_bytes(rec[32 * k:32 * k + 32], "little")
            rec = set_word(rec, k, w ^ (1 << rng.randrange(254)))
        elif kind == 3:
            rec = shift_record(rec, torsion[rng.randrange(3)])
        elif kind == 4:
            j = rng.randrange(6)
            w0 = int.from_bytes(rec[:32], "little")
            if j == 0:
                rec = set_word(rec, 0, (R + rng.randrange(1 << 250)) % (1 << 254) | (w0 >> 255 << 255))
            elif j == 1:
                rec = set_word(rec, 0, w0 | 1 << 254)
            elif j == 2:
                rec = set_word(rec, 1 + rng.randrange(4), R + rng.randrange(1 << 250))
            elif j == 3:
                cm = R + rng.randrange(1 << 250)
            elif j == 4:
                rec = set_word(rec, 0, bad_x)
            else:
                T = torsion[rng.randrange(3)]
                rec = set_word(rec, 0, T[0] | (T[1] & 1) << 255)
        recs.append(rec)
        cms.append(cm)
    return recs, cms


# ---- CPU: the spec ---------------------------------------------------------------------------------------------------------
def test_spec_reproduces_golden_vectors():
    keys = [int(v) for v in GOLD["view_keys"]]
    assert [list(N.public_key(v)) for v in keys] == [[int(x), o] for x, o in GOLD["public_keys"]]
    assert [N.public_key(v) for v in keys] == [bjj.to_pub(v) for v in keys]
    pks, notes, es, enc = golden_encryptions()
    for pk, note, e, x in zip(pks, notes, es, enc):
        st, rec, cm = N.encrypt(pk, note, e)
        assert (st, rec.hex(), str(cm)) == (x["status"], x["record"], x["commitment"])
    assert {x["status"] for x in enc} == {1, 2, 3}
    recs, cms, owners, plain = golden_scan()
    assert N.scan(keys, recs, cms) == (owners, plain)
    assert owners.count(N.MALFORMED) == 6 and N.NOT_OWNED in owners and 0 in owners and 1 in owners


def test_spec_round_trip_wrong_key_and_tampering():
    rng = random.Random(7)
    for _ in range(6):
        v = rng.randrange(1, R)
        note = rand_note(rng)
        st, rec, cm = N.encrypt(N.public_key(v), note, rng.randrange(1, R))
        assert st == N.ENC_OK and cm == N.commitment(note)
        assert N.decrypt_or_none(v, rec, cm) == note
        assert N.decrypt_or_none(rng.randrange(1, R), rec, cm) is None
        for k in range(5):                               # every word, and the commitment
            w = int.from_bytes(rec[32 * k:32 * k + 32], "little")
            bad = set_word(rec, k, w ^ (1 << rng.randrange(256)))
            assert N.decrypt_or_none(v, bad, cm) is None
            assert N.scan([v], [bad], [cm])[0][0] in (N.NOT_OWNED, N.MALFORMED)
        assert N.scan([v], [rec], [cm ^ 1])[0][0] in (N.NOT_OWNED, N.MALFORMED)


def test_spec_torsion_shifted_ephemeral_still_decrypts():
    """E + T for T of order 2, 4 and 8 (l P for a point P outside the subgroup) gives the same shared point: 8 (E + T) = 8 E."""
    T2, T4, T8 = torsion_points()
    for T, order in ((T2, 2), (T4, 4), (T8, 8)):
        assert N.mul(T, order) == N.IDENTITY and N.mul(T, order // 2) != N.IDENTITY
    rng = random.Random(8)
    v = rng.randrange(1, R)
    note = rand_note(rng)
    _, rec, cm = N.encrypt(N.public_key(v), note, rng.randrange(1, R))
    for T in (T2, T4, T8):
        shifted = shift_record(rec, T)
        assert shifted != rec and N.decrypt_or_none(v, shifted, cm) == note


def test_spec_keys_equal_mod_l_own_the_same_records():
    rng = random.Random(9)
    v = rng.randrange(1, R - L)
    assert N.public_key(v) == N.public_key(v + L)
    recs, cms = mixed_records(rng, [v], 24)
    o1, p1 = N.scan([v], recs, cms)
    o2, p2 = N.scan([v + L], recs, cms)
    assert o1 == o2 and p1 == p2 and 0 in o1
    assert N.scan([v + L, v], recs, cms)[0] == o1       # both own: the lower index
    for bad in (0, L, 7 * L, R):
        with pytest.raises(ValueError):
            N.public_key(bad)


# ---- CPU: the core of the kernels, compiled for the host ----------------------------------------------------------------------
@pytest.fixture(scope="module")
def h(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("notes") / "libnote_harness.so")      # the source tree may be read-only
    src = os.path.join(ROOT, "tests", "harness", "note_harness.cpp")
    subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-I" + os.path.join(ROOT, "owshen_b200", "csrc"), "-o", so, src],
                   check=True)
    return C.CDLL(so)


def h_encrypt(h, pks, notes, es):
    n = len(pks)
    am = (C.c_uint64 * n)(*[m[3] for m in notes])
    rec, cm, st = C.create_string_buffer(160 * n), C.create_string_buffer(32 * n), C.create_string_buffer(n)
    h.nh_encrypt(fr([p[0] for p in pks]), bytes(p[1] for p in pks), *[fr([m[k] for m in notes]) for k in range(3)], am, fr(es),
                 C.c_uint64(n), fr(bjj.BASE), rec, cm, st)
    return rec.raw, cm.raw, st.raw


def h_scan(h, keys, recs, cms, window):
    n = len(recs)
    owner, plain = (C.c_uint32 * n)(), C.create_string_buffer(128 * n)
    h.nh_scan(fr(keys), len(keys), b"".join(recs), fr(cms), C.c_uint64(n), window, owner, plain)
    return list(owner), words(plain.raw, 128)


def test_host_core_matches_golden_vectors(h):
    keys = [int(v) for v in GOLD["view_keys"]]
    px, odd = C.create_string_buffer(64), C.create_string_buffer(2)
    h.nh_public_keys(fr(keys), C.c_uint64(2), fr(bjj.BASE), px, odd)
    assert [[int.from_bytes(px.raw[32 * i:32 * i + 32], "little"), odd.raw[i]] for i in range(2)] == [[int(x), o] for x, o in GOLD["public_keys"]]
    pks, notes, es, enc = golden_encryptions()
    rec, cm, st = h_encrypt(h, pks, notes, es)
    assert list(st) == [x["status"] for x in enc]
    assert rec == b"".join(bytes.fromhex(x["record"]) for x in enc)
    assert cm == fr([int(x["commitment"]) for x in enc])
    recs, cms, owners, plain = golden_scan()
    for window in (0, 1):
        assert h_scan(h, keys, recs, cms, window) == (owners, plain)


def test_host_core_matches_spec_on_random_and_edge_records(h):
    rng = random.Random(10)
    keys = [rng.randrange(1, R) for _ in range(2)]
    pks = [N.public_key(keys[i % 2]) if i % 5 else N.public_key(rng.randrange(1, R)) for i in range(64)]
    edge_e = [1, L - 1, L, 2 * L, L + 1, R - 1, 0]
    es = edge_e + [rng.randrange(1, R) for _ in range(64 - len(edge_e))]
    notes = [rand_note(rng, [0, (1 << 64) - 1, None][i % 3]) for i in range(64)]
    notes[5] = (0, R - 1, 0, 0)
    rec, cm, st = h_encrypt(h, pks, notes, es)
    spec = [N.encrypt(p, m, e) for p, m, e in zip(pks, notes, es)]
    assert list(st) == [s[0] for s in spec] and rec == b"".join(s[1] for s in spec) and cm == fr([s[2] for s in spec])
    recs, cms = mixed_records(rng, keys, 240)
    recs += words(rec, 160)
    cms += [s[2] for s in spec]
    expect = N.scan(keys, recs, cms)
    assert {N.MALFORMED, N.NOT_OWNED, 0, 1} <= set(expect[0])
    for window in (0, 1):
        assert h_scan(h, keys, recs, cms, window) == expect


# ---- CPU: the transaction envelope ------------------------------------------------------------------------------------------
def test_shielded_transfer_envelope():
    rng = random.Random(11)
    proof, pub, recs = (bytes(rng.randrange(256) for _ in range(k)) for k in (256, 256, 320))
    msg = formats.shielded_transfer_to_rlp(proof, pub, recs)
    assert formats.shielded_transfer_from_rlp(msg) == (proof, pub, recs)
    for args in ((proof[:-1], pub, recs), (proof, pub + b"\0", recs), (proof, pub, recs[:160])):
        with pytest.raises(ValueError):
            formats.shielded_transfer_to_rlp(*args)
    items = [formats.SHIELDED_TRANSFER_KIND.encode(), proof] + words(pub, 32) + words(recs, 160)
    bad = [items[:-1], items + [b"x"], [b"shielded-withdraw"] + items[1:], items[:1] + [proof[:255]] + items[2:],
           items[:3] + [items[3][:31]] + items[4:], items[:-1] + [items[-1] + b"\0"], items[:5] + [[items[5]]] + items[6:]]
    for it in bad:
        with pytest.raises(ValueError, match="Invalid tx!"):
            formats.shielded_transfer_from_rlp(formats.rlp_encode(it))
    for junk in (b"", msg[:-1], msg + b"\0", formats.rlp_encode(b"shielded-transfer")):
        with pytest.raises(ValueError):
            formats.shielded_transfer_from_rlp(junk)
    wmsg = formats.shielded_withdraw_to_rlp(proof, pub[:96])
    with pytest.raises(ValueError, match="Invalid tx!"):
        formats.shielded_transfer_from_rlp(wmsg)


# ---- GPU -------------------------------------------------------------------------------------------------------------------
def gpu_encrypt(ctx, pks, notes, es):
    return ctx.note_encrypt(fr([p[0] for p in pks]), bytes(p[1] for p in pks), *[fr([m[k] for m in notes]) for k in range(3)],
                            [m[3] for m in notes], fr(es))


@pytest.mark.gpu
def test_gpu_public_keys_and_encrypt_match_spec(ctx):
    keys = [int(v) for v in GOLD["view_keys"]]
    rng = random.Random(12)
    keys += [rng.randrange(1, R) for _ in range(30)] + [1, L - 1, L + 1, R - 1]
    px, odd = ctx.note_public_keys(fr(keys))
    spec = [N.public_key(v) for v in keys]
    assert px == fr([p[0] for p in spec]) and list(odd) == [p[1] for p in spec]
    pks, notes, es, enc = golden_encryptions()
    rec, cm, st = gpu_encrypt(ctx, pks, notes, es)
    assert list(st) == [x["status"] for x in enc] and rec == b"".join(bytes.fromhex(x["record"]) for x in enc)
    assert cm == fr([int(x["commitment"]) for x in enc])
    # 256 notes: edge ephemerals, amounts and fields, foreign and refused keys
    n = 256
    bad_x = non_decompressing_x()
    pks = [spec[i % len(spec)] for i in range(n)]
    pks[3], pks[4], pks[5] = (bad_x, 0), (0, 1), (0, 0)
    es = [1, L - 1, L, 2 * L, L + 1, R - 1, 0] + [rng.randrange(1, R) for _ in range(n - 7)]
    notes = [rand_note(rng, [0, (1 << 64) - 1, None][i % 3]) for i in range(n)]
    notes[7], notes[8] = (0, R - 1, 0, 0), (R - 1, 0, R - 1, (1 << 64) - 1)
    rec, cm, st = gpu_encrypt(ctx, pks, notes, es)
    sp = [N.encrypt(p, m, e) for p, m, e in zip(pks, notes, es)]
    assert list(st) == [s[0] for s in sp] and {1, 2, 3} <= set(st)
    assert rec == b"".join(s[1] for s in sp) and cm == fr([s[2] for s in sp])


@pytest.mark.gpu
def test_gpu_scan_matches_spec(ctx):
    keys = [int(v) for v in GOLD["view_keys"]]
    recs, cms, owners, plain = golden_scan()
    got_o, got_p = ctx.note_scan(fr(keys), b"".join(recs), fr(cms))
    assert got_o == owners and words(got_p, 128) == plain
    rng = random.Random(13)
    base = rng.randrange(1, R - L)
    for k, n in ((1, 256), (3, 256), (17, 64)):
        ks = [rng.randrange(1, R) for _ in range(k)]
        if k == 17:
            ks[4], ks[11] = base + L, base                   # v + l at the lower index owns what v owns
        recs, cms = mixed_records(rng, ks, n)
        expect = N.scan(ks, recs, cms)
        got_o, got_p = ctx.note_scan(fr(ks), b"".join(recs), fr(cms))
        assert got_o == expect[0], k
        assert words(got_p, 128) == expect[1], k
        if k == 17:
            assert 4 in got_o and 11 not in got_o


@pytest.mark.gpu
def test_gpu_dev_entry_points_and_argument_errors(ctx):
    import torch
    rng = random.Random(14)
    keys = [rng.randrange(1, R) for _ in range(3)]
    pks = [N.public_key(keys[i % 3]) for i in range(40)]
    notes = [rand_note(rng) for _ in range(40)]
    es = [rng.randrange(1, R) for _ in range(40)]
    rec, cm, st = gpu_encrypt(ctx, pks, notes, es)
    dev = torch.device("cuda", ctx.device)
    u8 = lambda b: torch.frombuffer(bytearray(b), dtype=torch.uint8).to(dev)
    ins = [u8(fr([p[0] for p in pks])), u8(bytes(p[1] for p in pks))] + [u8(fr([m[k] for m in notes])) for k in range(3)]
    ins += [u8(struct.pack("<40Q", *[m[3] for m in notes])), u8(fr(es))]
    d_rec, d_cm, d_st = (torch.zeros(k * 40, dtype=torch.uint8, device=dev) for k in (160, 32, 1))
    ctx.note_encrypt_dev(*ins, 40, d_rec, d_cm, d_st)
    ctx.sync()
    assert (bytes(d_rec.cpu().numpy()), bytes(d_cm.cpu().numpy()), bytes(d_st.cpu().numpy())) == (rec, cm, st)
    owners, plain = ctx.note_scan(fr(keys), rec, cm)
    d_owner = torch.zeros(40, dtype=torch.int32, device=dev)
    d_plain = torch.zeros(128 * 40, dtype=torch.uint8, device=dev)
    ctx.note_scan_dev(fr(keys), d_rec, d_cm, 40, d_owner, d_plain)
    ctx.sync()
    assert [x & 0xFFFFFFFF for x in d_owner.cpu().tolist()] == owners == [i % 3 for i in range(40)]
    assert bytes(d_plain.cpu().numpy()) == plain
    # lengths
    with pytest.raises(ValueError):
        ctx.note_scan(fr(keys), rec[:-1], cm)
    with pytest.raises(ValueError):
        ctx.note_scan(fr(keys), rec, cm[:-32])
    with pytest.raises(ValueError):
        ctx.note_scan(fr(keys)[:-1], rec, cm)
    with pytest.raises(ValueError):
        ctx.note_public_keys(fr(keys)[:-1])
    with pytest.raises(ValueError):
        ctx.note_encrypt(fr([p[0] for p in pks]), bytes(p[1] for p in pks), fr([1] * 40), fr([1] * 40), fr([1] * 39), [1] * 40)
    with pytest.raises(ValueError):
        ctx.note_encrypt(fr([p[0] for p in pks]), bytes(p[1] for p in pks), fr([1] * 40), fr([1] * 40), fr([1] * 40), [1] * 39)
    # bad view keys: the caller's error, with the documented codes
    for bad, code in ((R, -2), ((1 << 256) - 1, -2), (0, -1), (L, -1), (5 * L, -1)):
        with pytest.raises(ob.OwshenB200Error) as e:
            ctx.note_scan(fr(keys[:1]) + bad.to_bytes(32, "little"), rec, cm)
        assert e.value.code == code, bad
        with pytest.raises(ob.OwshenB200Error) as e:
            ctx.note_public_keys(bad.to_bytes(32, "little"))
        assert e.value.code == code, bad
    # drawn ephemerals: a fresh encryption that still decrypts
    rec2, cm2, st2 = ctx.note_encrypt(fr([p[0] for p in pks]), bytes(p[1] for p in pks), *[fr([m[k] for m in notes]) for k in range(3)],
                                      [m[3] for m in notes])
    assert list(st2) == [1] * 40 and cm2 == cm and rec2 != rec
    assert ctx.note_scan(fr(keys), rec2, cm2) == (owners, plain)


@pytest.mark.gpu
def test_gpu_scan_at_scale(ctx):
    """2^20 records from the GPU encryption, about 1 in 1 000 to one of 8 scanning keys, the rest to 64 foreign keys."""
    n = 1 << 20
    rng = random.Random(15)
    nrng = np.random.default_rng(15)
    keys = [rng.randrange(1, R) for _ in range(8)]
    foreign = [rng.randrange(1, R) for _ in range(64)]
    px, odd = ctx.note_public_keys(fr(keys + foreign))
    px = np.frombuffer(px, dtype=np.uint8).reshape(72, 32)
    odd = np.frombuffer(odd, dtype=np.uint8)
    dest = nrng.integers(8, 72, size=n)
    planted = np.sort(nrng.choice(n, size=n // 1000, replace=False))
    dest[planted] = nrng.integers(0, 8, size=len(planted))

    def rand_fr(bits_top):                                   # n canonical elements below 2^(248 + bits_top)
        a = nrng.integers(0, 256, size=(n, 32), dtype=np.uint8)
        a[:, 31] &= (1 << bits_top) - 1
        return a

    nul, sec, tok = rand_fr(5), rand_fr(5), rand_fr(5)
    eph = rand_fr(2)                                          # < 2^250 < l
    eph[:, 0] |= 1                                            # nonzero
    amounts = nrng.integers(0, 1 << 63, size=n, dtype=np.uint64)
    rec, cm, st = ctx.note_encrypt(px[dest].tobytes(), odd[dest].tobytes(), nul.tobytes(), sec.tobytes(), tok.tobytes(),
                                   amounts.tobytes(), eph.tobytes())
    assert st == b"\x01" * n
    owners, plain = ctx.note_scan(fr(keys), rec, cm)
    o = np.array(owners, dtype=np.uint64)
    flagged = np.nonzero(o != N.NOT_OWNED)[0]
    assert np.array_equal(flagged, planted)
    assert np.array_equal(o[planted], dest[planted].astype(np.uint64))
    p = np.frombuffer(plain, dtype=np.uint8).reshape(n, 4, 32)
    am = np.zeros((n, 32), dtype=np.uint8)
    am[:, :8] = amounts.view(np.uint8).reshape(n, 8)
    assert np.array_equal(p[planted], np.stack([nul, sec, tok, am], axis=1)[planted])
    assert not p[o == N.NOT_OWNED].any()
    sample = sorted(set(rng.sample(range(n), 48)) | set(planted[:16].tolist()))
    spec = N.scan(keys, [rec[160 * i:160 * i + 160] for i in sample], [int.from_bytes(cm[32 * i:32 * i + 32], "little") for i in sample])
    assert [owners[i] for i in sample] == spec[0]
    assert [plain[128 * i:128 * i + 128] for i in sample] == spec[1]
    assert ctx.note_scan(fr(keys), rec, cm)[0] == owners


@pytest.mark.gpu
def test_transfer_outputs_delivered_and_spent(ctx):
    """A deposit's outputs go to A and B as encrypted records, A finds its note by scanning, spends it in a withdrawal with
    change encrypted back to A, and finds the change; every proof verifies."""
    from tests.test_transfer import pack, row
    rng = random.Random(16)
    depth = 2
    tw = [rng.randrange(1, R) for _ in range(5)]
    pk, vk = ob.setup_transfer(ctx, depth, *tw)
    PK = ob.ProvingKey(ctx, pk)
    tree = ob.MerkleTree(ctx, depth)
    vA, vB = rng.randrange(1, R), rng.randrange(1, R)
    pk_x, pk_odd = ctx.note_public_keys(fr([vA, vB]))
    to_x, to_odd = words(pk_x, 32), list(pk_odd)          # output 0 to A, output 1 to B
    token = rng.randrange(1 << 160)
    as_int = lambda b: int.from_bytes(b, "little")
    chain = []                                   # (records, commitments) in leaf order

    def prove_one(r):
        proofs, pub = PK.prove_transfer(*pack([r]), cport.frs([rng.randrange(R) for _ in range(2)]))
        assert ob.verify(vk, pub, proofs)
        return proofs, pub

    def deliver(outs, to_x, to_odd, pub):
        recs, cms, st = ctx.note_encrypt(b"".join(to_x), bytes(to_odd), *[fr([o[k] for o in outs]) for k in range(2)],
                                         fr([token, token]), [o[2] for o in outs])
        assert st == b"\x01\x01" and cms == pub[192:256]        # the proof's out_commitment public inputs
        chain.extend(zip(words(recs, 160), words(cms, 32)))
        return recs

    def decoys(k):
        vs = [rng.randrange(1, R) for _ in range(k)]
        x, o = ctx.note_public_keys(fr(vs))
        recs, cms, _ = ctx.note_encrypt(x, o, *[fr([rng.randrange(R) for _ in range(k)]) for _ in range(3)], [5] * k)
        return list(zip(words(recs, 160), words(cms, 32)))

    def scan_a():
        recs = chain + decoys(5)
        owners, plain = ctx.note_scan(fr([vA]), b"".join(r for r, _ in recs), b"".join(c for _, c in recs))
        return [i for i, o in enumerate(owners) if o == 0], words(plain, 128)

    try:
        dummy = [(rng.randrange(R), rng.randrange(R), 0, [0] * depth, 0) for _ in range(2)]
        d_out = [(rng.randrange(R), rng.randrange(R), 1000), (rng.randrange(R), rng.randrange(R), 500)]
        proofs, pub = prove_one(row(as_int(tree.root()), token, rng.randrange(1 << 160), dummy, d_out))
        recs = deliver(d_out, to_x, to_odd, pub)
        assert formats.shielded_transfer_from_rlp(formats.shielded_transfer_to_rlp(proofs, pub, recs)) == (proofs, pub, recs)
        idx = tree.insert_batch([pub[192:224], pub[224:256]])
        assert list(idx) == [0, 1]
        mine, plain = scan_a()
        assert mine == [0] and plain[0] == fr([d_out[0][0], d_out[0][1], token, 1000])
        # A withdraws 700 to a recipient; 300 change back to A, a zero-value second output to B
        sib, bits = tree.paths([0])
        a_in = (d_out[0][0], d_out[0][1], 1000, cport.unfr(sib), bits[0])
        w_out = [(rng.randrange(R), rng.randrange(R), 300), (rng.randrange(R), rng.randrange(R), 0)]
        proofs, pub = prove_one(row(as_int(tree.root()), token, rng.randrange(1 << 160),
                                    [a_in, (rng.randrange(R), rng.randrange(R), 0, [0] * depth, 0)], w_out))
        assert as_int(pub[32:64]) == R - 700
        deliver(w_out, to_x, to_odd, pub)
        tree.insert_batch([pub[192:224], pub[224:256]])
        mine, plain = scan_a()
        assert mine == [0, 2] and plain[2] == fr([w_out[0][0], w_out[0][1], token, 300])
    finally:
        PK.close()
