"""Generates tests/golden/note_vectors.json from the spec of encrypted notes (oracle/notes.py) with a fixed seed: two view
keys and their addresses, encryptions covering edge amounts (0, 2^64 - 1), field edges (0, r - 1), ephemerals 1, l - 1 and
>= l, every refusal status, and a scan of the records plus one malformed record of each kind, a foreign record, a tampered
one and torsion-shifted ones under both keys.
Run from the repo root:  python -m tests.golden.gen_note_golden
"""
import json
import os
import random

from oracle import notes as N
from oracle.bn254 import R

HERE = os.path.dirname(os.path.abspath(__file__))
L = N.L


def non_decompressing_x():
    """The smallest x >= 2 that is no curve point's x (the square root fails)."""
    x = 2
    while N.decompress_or_none(x, 0) is not None:
        x += 1
    return x


def torsion_points():
    """Points of order 2, 4 and 8: l P and its doublings, for the first decompressed P with 4 l P != O."""
    x = 2
    while True:
        P = N.decompress_or_none(x, 0)
        if P is not None:
            t8 = N.mul(P, L)
            if N.mul(t8, 4) != N.IDENTITY:
                return [N.mul(t8, 4), N.mul(t8, 2), t8]
        x += 1


def shift_record(record, T):
    """The record with E replaced by E + T (same ciphertext)."""
    w0 = int.from_bytes(record[:32], "little")
    x, odd = w0 & ((1 << 255) - 1), w0 >> 255
    E2 = N.add(N.bjj.decompress((x, odd)), T)
    return N.encode_record(E2[0], E2[1] & 1, []) + record[32:]


def set_word(record, i, value):
    return record[:32 * i] + value.to_bytes(32, "little") + record[32 * i + 32:]


def main():
    rng = random.Random(20261017)
    keys = [rng.randrange(1, R) for _ in range(2)]
    pks = [N.public_key(v) for v in keys]
    cases = []                                   # (pk, note, e)
    edge_notes = [(0, R - 1, 0, 0), (R - 1, 0, R - 1, (1 << 64) - 1), (rng.randrange(R), rng.randrange(R), 1, 1)]
    for j, note in enumerate(edge_notes):
        cases.append((pks[j % 2], note, rng.randrange(1, R)))
    for e in (1, L - 1, L, L + 1, 2 * L + 7, R - 1, 0):
        cases.append((pks[len(cases) % 2], (rng.randrange(R), rng.randrange(R), rng.randrange(R), rng.randrange(1 << 64)), e))
    foreign = N.public_key(rng.randrange(1, R))
    cases.append((foreign, (rng.randrange(R),) * 3 + (5,), rng.randrange(1, R)))
    bad_x = non_decompressing_x()
    for pk in ((bad_x, 0), (0, 1), (0, 0)):      # no point; the identity; the point of order 2
        cases.append((pk, (1, 2, 3, 4), rng.randrange(1, R)))
    enc = []
    for pk, note, e in cases:
        st, rec, cm = N.encrypt(pk, note, e)
        enc.append(dict(pk_x=str(pk[0]), pk_odd=pk[1], note=[str(x) for x in note], e=str(e), status=st, record=rec.hex(), commitment=str(cm)))
    good = [(bytes.fromhex(x["record"]), int(x["commitment"])) for x in enc if x["status"] == N.ENC_OK]
    rec0, cm0 = good[0]
    T2, T4, T8 = torsion_points()
    scan_recs = list(good)
    scan_recs += [(shift_record(rec0, T), cm0) for T in (T2, T4, T8)]
    scan_recs.append((set_word(rec0, 2, int.from_bytes(rec0[64:96], "little") ^ 1), cm0))       # tampered: not owned
    w0 = int.from_bytes(rec0[:32], "little")
    scan_recs += [
        (set_word(rec0, 0, R | (w0 >> 255 << 255)), cm0),         # x >= r
        (set_word(rec0, 0, w0 | 1 << 254), cm0),                  # bit 254 set
        (set_word(rec0, 3, R), cm0),                              # c_2 >= r
        (rec0, R),                                                # commitment >= r
        (set_word(rec0, 0, bad_x), cm0),                          # E does not decompress
        (set_word(rec0, 0, 0), cm0),                              # E of order 2: 8 E = O
    ]
    owners, plain = N.scan(keys, [r for r, _ in scan_recs], [c for _, c in scan_recs])
    out = dict(view_keys=[str(v) for v in keys], public_keys=[[str(x), o] for x, o in pks], encryptions=enc,
               scan=dict(records=[r.hex() for r, _ in scan_recs], commitments=[str(c) for _, c in scan_recs], owners=owners,
                         plaintexts=[p.hex() for p in plain]))
    with open(os.path.join(HERE, "note_vectors.json"), "w") as f:
        json.dump(out, f, indent=1)
    print("wrote note_vectors.json", len(enc), "encryptions,", len(scan_recs), "scanned records, owners", owners)


if __name__ == "__main__":
    main()
