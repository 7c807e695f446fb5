"""Shared test helpers: serialisation of oracle keys into the product's blob formats, input generators."""
import random
import struct

from oracle import bn254 as bn
from oracle import cport

R, P = bn.R, bn.P


def vk_blob(vkb: dict, n_pub: int = 3) -> bytes:
    return (b"OGVK" + struct.pack("<II", 1, n_pub) + vkb["alpha1"] + vkb["beta2"] + vkb["gamma2"] + vkb["delta2"] + vkb["ic"])


def pk_blob(cs, pkb: dict, depth: int) -> bytes:
    blob = b"OGPK" + struct.pack("<IIIIII", 1, depth, cs.n_constraints, cs.n_vars, cs.n_pub, pkb["log_m"])
    blob += pkb["alpha1"] + pkb["beta1"] + pkb["beta2"] + pkb["delta1"] + pkb["delta2"]
    blob += pkb["a"] + pkb["b1"] + pkb["b2"] + pkb["l"] + pkb["h"]
    for m in "AB":
        ptr, idx, val = cs.csr(m)
        blob += struct.pack("<I", len(idx)) + struct.pack(f"<{len(ptr)}I", *ptr) + struct.pack(f"<{len(idx)}I", *idx) + cport.frs(val)
    return blob


_KEYS32 = None


def withdraw_keys32(ctx):
    """Depth-32 withdraw keys from the library's setup and from the oracle's: (pk, vk, r1cs, oracle pk bytes, oracle vk bytes).
    Made once per process, so every module that proves at depth 32 shares one setup."""
    global _KEYS32
    if _KEYS32 is None:
        import owshen_b200 as ob
        from oracle import withdraw_circuit as wc
        rng = random.Random(10)
        tw = [rng.randrange(1, R) for _ in range(5)]
        pk, vk = ob.setup_withdraw(ctx, 32, *tw)
        cs = wc.build_r1cs(32)
        pkb, vkb = cport.setup_bytes(cs, *tw)
        _KEYS32 = (pk, vk, cs, pkb, vkb)
    return _KEYS32


def rand_inputs(rng: random.Random, batch: int, depth: int):
    nul = cport.frs([rng.randrange(R) for _ in range(batch)])
    sec = cport.frs([rng.randrange(R) for _ in range(batch)])
    rec = cport.frs([rng.randrange(1 << 160) for _ in range(batch)])
    sib = cport.frs([rng.randrange(R) for _ in range(batch * depth)])
    bits = [rng.randrange(1 << depth) for _ in range(batch)]
    return nul, sec, rec, sib, bits


def rand_g1(rng: random.Random, n: int) -> bytes:
    return cport.g1_fixed_mul_batch(bn.g1_to_bytes(bn.G1_GEN), cport.frs([rng.randrange(R) for _ in range(n)]))


def rand_g2(rng: random.Random, n: int) -> bytes:
    return cport.g2_fixed_mul_batch(bn.g2_to_bytes(bn.G2_GEN), cport.frs([rng.randrange(R) for _ in range(n)]))


def rand_fr_bytes(rng: random.Random, n: int) -> bytes:
    """n uniform 248-bit values (always canonical), fast to generate in bulk."""
    raw = rng.randbytes(31 * n)
    return b"".join(raw[31 * i:31 * i + 31] + b"\0" for i in range(n))
