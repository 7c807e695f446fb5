"""Encrypted note delivery: the frozen spec of BabyJubJub note encryption and note scanning (DESIGN.md section 3,
"Encrypted notes").  Not in the reference; built on its curve (oracle/babyjubjub.py) and on circomlib's MiMC7
(oracle/mimc7.py).

A wallet's view key v (canonical Fr, v mod l != 0) has the public key V = compress(v BASE), exactly `to_pub`.  A sender
encrypts a note m = (nullifier, secret, token, amount < 2^64) to V with an ephemeral scalar e (e mod l != 0):
    V' = 8 V (refused if O),  E = e BASE,  S = affine(e V'),  k = MultiMiMC7([S.x, S.y], 0),
    c_i = m_i + MiMC7(i, k)  for i = 0..3.
The 160-byte record is  E.x | parity(E.y) << 255  followed by c_0..c_3 (32-byte little-endian words).  The receiver
computes S = v (8 E), which equals e V' because 8 E and V' lie in the prime-order subgroup; the note is owned iff
MultiMiMC7(m, 0) equals the transfer proof's output commitment and the amount fits 64 bits.  Clearing the cofactor of E
makes S independent of any low-order part a sender adds to E.
"""
from . import babyjubjub as bjj
from . import mimc7
from .bn254 import R

L = bjj.ORDER // 8                 # the prime order of BASE
RECORD_BYTES = 160
PLAINTEXT_BYTES = 128
NOT_OWNED = 0xFFFFFFFF
MALFORMED = 0xFFFFFFFE
ENC_OK, ENC_BAD_KEY, ENC_BAD_EPHEMERAL = 1, 2, 3
IDENTITY = (0, 1)


# complete projective formulas of the curve (the reference's, babyjubjub.p_add without its equality test, which the
# unified addition does not need): fast enough to scan hundreds of records in tests
def _padd(p, q):
    X1, Y1, Z1 = p
    X2, Y2, Z2 = q
    a = Z1 * Z2 % R; b = a * a % R; c = X1 * X2 % R; d = Y1 * Y2 % R
    e = bjj.D * c % R * d % R; f = (b - e) % R; g = (b + e) % R
    return (a * f % R * ((X1 + Y1) * (X2 + Y2) - c - d) % R, a * g % R * (d - bjj.A * c) % R, f * g % R)


def mul(p, k):
    """k p for an affine point p and any integer k >= 0 (no reduction of k), as an affine point."""
    acc = (0, 1, 1)
    pp = (p[0], p[1], 1)
    for i in range(k.bit_length() - 1, -1, -1):
        acc = _padd(acc, acc)
        if (k >> i) & 1:
            acc = _padd(acc, pp)
    zi = pow(acc[2], -1, R)
    return (acc[0] * zi % R, acc[1] * zi % R)


def add(p, q):
    return _affine(_padd((p[0], p[1], 1), (q[0], q[1], 1)))


def _affine(p):
    zi = pow(p[2], -1, R)
    return (p[0] * zi % R, p[1] * zi % R)


def clear_cofactor(p):
    return mul(p, 8)


def decompress_or_none(x, odd):
    try:
        return bjj.decompress((x, odd))
    except bjj.CannotInvert:
        return None


def valid_view_key(v):
    return 0 <= v < R and v % L != 0


def public_key(v):
    """-> (x, parity of y): the compressed point v BASE, i.e. PrivateKey::to_pub."""
    if not valid_view_key(v):
        raise ValueError("view key must be canonical and nonzero mod l")
    return bjj.compress(mul(bjj.BASE, v))


def commitment(note):
    return mimc7.multi_hash(list(note), 0)


def _key(s):
    return mimc7.multi_hash([s[0], s[1]], 0)


def _pad(i, k):
    return mimc7.mimc7_hash(i, k)


def encode_record(ex, e_odd, cs):
    w0 = ex | (e_odd << 255)
    return w0.to_bytes(32, "little") + b"".join(c.to_bytes(32, "little") for c in cs)


def encrypt(pk, note, e):
    """-> (status, record, commitment); status ENC_OK, ENC_BAD_KEY (V does not decompress or 8 V = O) or
    ENC_BAD_EPHEMERAL (e = 0 mod l).  A refused note has an all-zero record and commitment."""
    nullifier, secret, token, amount = note
    assert all(0 <= x < R for x in (nullifier, secret, token, pk[0], e)) and 0 <= amount < 1 << 64
    fail = lambda st: (st, bytes(RECORD_BYTES), 0)
    V = decompress_or_none(*pk)
    if V is None:
        return fail(ENC_BAD_KEY)
    Vp = clear_cofactor(V)
    if Vp == IDENTITY:
        return fail(ENC_BAD_KEY)
    if e % L == 0:
        return fail(ENC_BAD_EPHEMERAL)
    E = mul(bjj.BASE, e)
    k = _key(mul(Vp, e))
    cs = [(m + _pad(i, k)) % R for i, m in enumerate(note)]
    return ENC_OK, encode_record(E[0], E[1] & 1, cs), commitment(note)


def prepare(record, cm):
    """The per-record half of a scan: 8 E and the four ciphertext words, or None when the record is malformed."""
    assert len(record) == RECORD_BYTES
    w = [int.from_bytes(record[32 * i:32 * i + 32], "little") for i in range(5)]
    x, odd = w[0] & ((1 << 255) - 1), w[0] >> 255
    if x >= R or any(c >= R for c in w[1:]) or cm >= R:      # x >= R covers bit 254
        return None
    E = decompress_or_none(x, odd)
    if E is None:
        return None
    Ep = clear_cofactor(E)
    if Ep == IDENTITY:
        return None
    return Ep, w[1:]


def decrypt_prepared(v, prepared, cm):
    Ep, cs = prepared
    k = _key(mul(Ep, v))
    m = [(c - _pad(i, k)) % R for i, c in enumerate(cs)]
    if m[3] >= 1 << 64 or commitment(m) != cm:
        return None
    return tuple(m)


def decrypt_or_none(v, record, cm):
    """The note (nullifier, secret, token, amount) when view key v owns the record, else None (also when malformed)."""
    p = prepare(record, cm)
    return None if p is None else decrypt_prepared(v, p, cm)


def scan(view_keys, records, commitments):
    """-> (owners, plaintexts): per record the lowest index of a key that owns it, NOT_OWNED or MALFORMED, and its
    note as four 32-byte words (all zero unless owned)."""
    owners, plain = [], []
    for rec, cm in zip(records, commitments):
        p = prepare(rec, cm)
        owner, note = (MALFORMED, None) if p is None else (NOT_OWNED, None)
        if p is not None:
            for j, v in enumerate(view_keys):
                note = decrypt_prepared(v, p, cm)
                if note is not None:
                    owner = j
                    break
        owners.append(owner)
        plain.append(bytes(PLAINTEXT_BYTES) if note is None else b"".join(x.to_bytes(32, "little") for x in note))
    return owners, plain
