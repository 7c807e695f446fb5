"""Proof / verifying-key encodings for consumers outside this library (SURVEY.md section 8f.1): the EVM
precompile layout of EIP-197 (what a Solidity Groth16 verifier next to
/root/reference/contracts/src/Owshen.sol:66-78 would take as calldata) and snarkjs-style JSON.
Pure byte shuffling of the library's own 256-byte proofs and OGVK blobs -- no arithmetic happens here.

Library layout (include/owshen_b200.h): little-endian 32-byte coordinates, G2 = x.c0 || x.c1 || y.c0 || y.c1.
EIP-197 / Solidity: big-endian 32-byte words, G2 = x.c1 || x.c0 || y.c1 || y.c0 (imaginary part first)."""
import json
import struct


def _ints(b: bytes):
    return [int.from_bytes(b[i:i + 32], "little") for i in range(0, len(b), 32)]


def _be(x: int) -> bytes:
    return x.to_bytes(32, "big")


def proof_points(proof: bytes):
    """(A, B, C) as integer coordinates: A = (x, y), B = ((x0, x1), (y0, y1)), C = (x, y)."""
    assert len(proof) == 256
    v = _ints(proof)
    return (v[0], v[1]), ((v[2], v[3]), (v[4], v[5])), (v[6], v[7])


def proof_to_eip197(proof: bytes) -> bytes:
    """a[2] || b[2][2] || c[2] as 8 big-endian words, the argument order of the usual Solidity verifyProof."""
    (ax, ay), ((bx0, bx1), (by0, by1)), (cx, cy) = proof_points(proof)
    return b"".join(_be(x) for x in (ax, ay, bx1, bx0, by1, by0, cx, cy))


def proof_from_eip197(data: bytes) -> bytes:
    assert len(data) == 256
    w = [int.from_bytes(data[i:i + 32], "big") for i in range(0, 256, 32)]
    ax, ay, bx1, bx0, by1, by0, cx, cy = w
    return b"".join(x.to_bytes(32, "little") for x in (ax, ay, bx0, bx1, by0, by1, cx, cy))


def public_inputs_to_eip197(public_inputs: bytes) -> bytes:
    return b"".join(_be(x) for x in _ints(public_inputs))


def proof_to_snarkjs(proof: bytes) -> dict:
    (ax, ay), ((bx0, bx1), (by0, by1)), (cx, cy) = proof_points(proof)
    s = str
    return {"pi_a": [s(ax), s(ay), "1"], "pi_b": [[s(bx0), s(bx1)], [s(by0), s(by1)], ["1", "0"]],
            "pi_c": [s(cx), s(cy), "1"], "protocol": "groth16", "curve": "bn128"}


def parse_vk(vk: bytes) -> dict:
    """OGVK v1 blob -> integer coordinates."""
    assert vk[:4] == b"OGVK"
    ver, n_pub = struct.unpack("<II", vk[4:12])
    assert ver == 1 and len(vk) == 12 + 64 + 3 * 128 + 64 * (n_pub + 1)
    v = _ints(vk[12:])
    g2 = lambda o: ((v[o], v[o + 1]), (v[o + 2], v[o + 3]))
    ic = [(v[14 + 2 * i], v[15 + 2 * i]) for i in range(n_pub + 1)]
    return {"n_pub": n_pub, "alpha1": (v[0], v[1]), "beta2": g2(2), "gamma2": g2(6), "delta2": g2(10), "ic": ic}


def vk_to_snarkjs(vk: bytes) -> dict:
    p = parse_vk(vk)
    s = str
    g1 = lambda q: [s(q[0]), s(q[1]), "1"]
    g2 = lambda q: [[s(q[0][0]), s(q[0][1])], [s(q[1][0]), s(q[1][1])], ["1", "0"]]
    return {"protocol": "groth16", "curve": "bn128", "nPublic": p["n_pub"], "vk_alpha_1": g1(p["alpha1"]),
            "vk_beta_2": g2(p["beta2"]), "vk_gamma_2": g2(p["gamma2"]), "vk_delta_2": g2(p["delta2"]),
            "IC": [g1(q) for q in p["ic"]]}


def to_json(obj: dict) -> str:
    return json.dumps(obj, indent=1)


# ---- the node's transaction envelope (SURVEY.md section 8f.4) ------------------------------------------------------
# /root/reference/src/types/tx/custom.rs:214-256 wraps every custom message as an RLP list whose first item is the
# message kind as a string ("mint", "burn"), byte fields following as RLP strings, integers as little-endian byte
# vectors (custom.rs:40, `amount.as_le_bytes()`).  A shielded withdrawal carrying one of this library's proofs takes
# the same shape:   ["shielded-withdraw", proof (256 B), root, nullifier_hash, recipient (32 B LE each)].
# RLP itself is the Ethereum yellow-paper appendix B encoding (crate `rlp` 0.5.2 in the reference's Cargo.toml:13).

SHIELDED_WITHDRAW_KIND = "shielded-withdraw"
# A shielded transfer carries its proof, the statement's 8 public inputs and the two 160-byte encrypted note records of its
# outputs (out 0, then out 1; DESIGN.md section 3, "Encrypted notes"):
#     ["shielded-transfer", proof (256 B), 8 public inputs (32 B LE each), record 0, record 1 (160 B each)]
SHIELDED_TRANSFER_KIND = "shielded-transfer"
# A shielded labeled transfer (the owned labeled transfer statement) has a kind of its own and 9 public inputs; its records are
# the owned labeled notes of its outputs:
#     ["shielded-labeled-transfer", proof (256 B), 9 public inputs (32 B LE each), record 0, record 1 (160 B each)]
SHIELDED_LABELED_TRANSFER_KIND = "shielded-labeled-transfer"
# A shielded ragequit (the public exit of an owned labeled note) has a kind of its own, 6 public inputs and no records: it
# creates no note.
#     ["shielded-ragequit", proof (256 B), 6 public inputs (32 B LE each)]
SHIELDED_RAGEQUIT_KIND = "shielded-ragequit"


def rlp_encode(item) -> bytes:
    """RLP of bytes / str / list (nested).  Integers are not accepted: the reference passes them as LE byte vectors."""
    if isinstance(item, str):
        item = item.encode()
    if isinstance(item, (bytes, bytearray)):
        b = bytes(item)
        if len(b) == 1 and b[0] < 0x80:
            return b
        return _rlp_len(len(b), 0x80) + b
    if isinstance(item, (list, tuple)):
        body = b"".join(rlp_encode(x) for x in item)
        return _rlp_len(len(body), 0xC0) + body
    raise TypeError(f"rlp_encode: unsupported {type(item).__name__}")


def _rlp_len(n: int, base: int) -> bytes:
    if n < 56:
        return bytes([base + n])
    nb = n.to_bytes((n.bit_length() + 7) // 8, "big")
    return bytes([base + 55 + len(nb)]) + nb


def rlp_decode(data: bytes):
    """Inverse of rlp_encode (strings come back as bytes).  Rejects trailing bytes and non-minimal lengths, like the
    reference's decoder returning DecoderError (custom.rs:176-183 maps those to a rejected transaction)."""
    item, end = _rlp_item(bytes(data), 0)
    if end != len(data):
        raise ValueError("rlp: trailing bytes")
    return item


def _rlp_item(d: bytes, i: int):
    if i >= len(d):
        raise ValueError("rlp: truncated")
    t = d[i]
    if t < 0x80:
        return d[i:i + 1], i + 1
    is_list = t >= 0xC0
    base = 0xC0 if is_list else 0x80
    if t - base < 56:
        n, start = t - base, i + 1
        if not is_list and n == 1 and start < len(d) and d[start] < 0x80:
            raise ValueError("rlp: single byte below 0x80 must be encoded as itself")
    else:
        ln = t - base - 55
        if i + 1 + ln > len(d) or d[i + 1] == 0:
            raise ValueError("rlp: bad length prefix")
        n, start = int.from_bytes(d[i + 1:i + 1 + ln], "big"), i + 1 + ln
        if n < 56:
            raise ValueError("rlp: non-minimal length")
    if start + n > len(d):
        raise ValueError("rlp: truncated")
    if not is_list:
        return d[start:start + n], start + n
    out, j = [], start
    while j < start + n:
        x, j = _rlp_item(d, j)
        out.append(x)
    if j != start + n:
        raise ValueError("rlp: list overruns its length")
    return out, j


def shielded_withdraw_to_rlp(proof: bytes, public_inputs: bytes) -> bytes:
    """CustomTxMsg-shaped message for one withdraw proof: public_inputs = root || nullifier_hash || recipient (96 B,
    the `public_out` row of og_groth16_prove_withdraw)."""
    if len(proof) != 256 or len(public_inputs) != 96:
        raise ValueError("shielded_withdraw_to_rlp: proof must be 256 bytes, public inputs 96")
    return rlp_encode([SHIELDED_WITHDRAW_KIND, proof, public_inputs[0:32], public_inputs[32:64], public_inputs[64:96]])


def shielded_withdraw_from_rlp(msg: bytes):
    """-> (proof, public_inputs); raises ValueError on anything that is not a well-formed shielded-withdraw message
    (the reference's from_rlp answers `Err(anyhow!("Invalid tx!"))` for an unknown kind, custom.rs:253)."""
    item = rlp_decode(msg)
    if not isinstance(item, list) or len(item) != 5 or any(isinstance(x, list) for x in item):
        raise ValueError("Invalid tx!")
    kind, proof, root, nh, rcpt = item
    if kind != SHIELDED_WITHDRAW_KIND.encode() or len(proof) != 256 or any(len(x) != 32 for x in (root, nh, rcpt)):
        raise ValueError("Invalid tx!")
    return proof, root + nh + rcpt


def shielded_transfer_to_rlp(proof: bytes, public_inputs: bytes, records: bytes) -> bytes:
    """CustomTxMsg-shaped message for one transfer proof: public_inputs = the 8 inputs of og_groth16_prove_transfer's
    `public_out` row (256 B), records = the encrypted notes of output 0 and output 1 (2 x 160 B, og_note_encrypt)."""
    if len(proof) != 256 or len(public_inputs) != 256 or len(records) != 320:
        raise ValueError("shielded_transfer_to_rlp: proof must be 256 bytes, public inputs 256, records 320")
    return rlp_encode([SHIELDED_TRANSFER_KIND, proof] + [public_inputs[32 * i:32 * i + 32] for i in range(8)]
                      + [records[0:160], records[160:320]])


def shielded_transfer_from_rlp(msg: bytes):
    """-> (proof, public_inputs, records); raises ValueError("Invalid tx!") on anything that is not a well-formed
    shielded-transfer message."""
    item = rlp_decode(msg)
    if not isinstance(item, list) or len(item) != 12 or any(isinstance(x, list) for x in item):
        raise ValueError("Invalid tx!")
    kind, proof, pub, recs = item[0], item[1], item[2:10], item[10:12]
    if kind != SHIELDED_TRANSFER_KIND.encode() or len(proof) != 256 or any(len(x) != 32 for x in pub) or any(len(r) != 160 for r in recs):
        raise ValueError("Invalid tx!")
    return proof, b"".join(pub), b"".join(recs)


def shielded_labeled_transfer_to_rlp(proof: bytes, public_inputs: bytes, records: bytes) -> bytes:
    """CustomTxMsg-shaped message for one owned labeled transfer proof: public_inputs = the 9 inputs of
    og_groth16_prove_owned_labeled_transfer's `public_out` row (288 B), records = the encrypted notes of output 0 and output 1
    (2 x 160 B, og_owned_labeled_note_encrypt)."""
    if len(proof) != 256 or len(public_inputs) != 288 or len(records) != 320:
        raise ValueError("shielded_labeled_transfer_to_rlp: proof must be 256 bytes, public inputs 288, records 320")
    return rlp_encode([SHIELDED_LABELED_TRANSFER_KIND, proof] + [public_inputs[32 * i:32 * i + 32] for i in range(9)]
                      + [records[0:160], records[160:320]])


def shielded_labeled_transfer_from_rlp(msg: bytes):
    """-> (proof, public_inputs, records); raises ValueError("Invalid tx!") on anything that is not a well-formed
    shielded-labeled-transfer message."""
    item = rlp_decode(msg)
    if not isinstance(item, list) or len(item) != 13 or any(isinstance(x, list) for x in item):
        raise ValueError("Invalid tx!")
    kind, proof, pub, recs = item[0], item[1], item[2:11], item[11:13]
    if (kind != SHIELDED_LABELED_TRANSFER_KIND.encode() or len(proof) != 256 or any(len(x) != 32 for x in pub)
            or any(len(r) != 160 for r in recs)):
        raise ValueError("Invalid tx!")
    return proof, b"".join(pub), b"".join(recs)


def shielded_ragequit_to_rlp(proof: bytes, public_inputs: bytes) -> bytes:
    """CustomTxMsg-shaped message for one ragequit proof: public_inputs = the 6 inputs of og_groth16_prove_ragequit's
    `public_out` row (192 B: root, token, amount, label, recipient, nullifier)."""
    if len(proof) != 256 or len(public_inputs) != 192:
        raise ValueError("shielded_ragequit_to_rlp: proof must be 256 bytes, public inputs 192")
    return rlp_encode([SHIELDED_RAGEQUIT_KIND, proof] + [public_inputs[32 * i:32 * i + 32] for i in range(6)])


def shielded_ragequit_from_rlp(msg: bytes):
    """-> (proof, public_inputs); raises ValueError("Invalid tx!") on anything that is not a well-formed shielded-ragequit
    message."""
    item = rlp_decode(msg)
    if not isinstance(item, list) or len(item) != 8 or any(isinstance(x, list) for x in item):
        raise ValueError("Invalid tx!")
    kind, proof, pub = item[0], item[1], item[2:8]
    if kind != SHIELDED_RAGEQUIT_KIND.encode() or len(proof) != 256 or any(len(x) != 32 for x in pub):
        raise ValueError("Invalid tx!")
    return proof, b"".join(pub)
