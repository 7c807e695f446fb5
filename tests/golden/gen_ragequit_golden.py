"""Generates tests/golden/ragequit_vectors.json from the spec (oracle/ragequit_circuit.py, oracle/groth16.py's setup exponents)
and the oracle's C port (fixed-base multiplications, prover) with a fixed seed: one depth-2 ragequit proof with every value
injected, its verifying key and the hashes of its proving-key queries and witness.
Run from the repo root after building the oracle (make -C oracle/cpu):  python -m tests.golden.gen_ragequit_golden
"""
import hashlib
import json
import os
import random

from oracle import bn254 as bn
from oracle import cport, mimc7
from oracle.ragequit_circuit import build_r1cs, note_leaf, spend_public_key, witness

R = bn.R
HERE = os.path.dirname(os.path.abspath(__file__))
DEPTH = 2


def main():
    rng = random.Random(20261019)
    cs = build_r1cs(DEPTH)
    tox = [rng.randrange(1, R) for _ in range(5)]
    pkb, vkb = cport.setup_bytes(cs, *tox)
    token, recipient = rng.randrange(1 << 160), rng.randrange(1 << 160)
    tree = mimc7.MerkleTree(DEPTH)
    tree.insert(rng.randrange(R))
    spend_key, blinding, amount = rng.randrange(R), rng.randrange(R), rng.randrange(1 << 64)
    label = tree.insert(note_leaf(spend_public_key(spend_key), blinding, token, amount, 1))     # the deposit at pool index 1
    sibs, bits = tree.path(label)
    path_bits = sum(x << l for l, x in enumerate(bits))
    r, s = rng.randrange(R), rng.randrange(R)
    w = witness(tree.root(), token, amount, label, recipient, spend_key, blinding, sibs, path_bits)
    assert cs.is_satisfied(w)
    wit = cport.frs(w)
    proof = cport.Prover(cs, pkb).prove(wit, r, s)
    out = dict(
        depth=DEPTH, toxic=[str(x) for x in tox], root=str(tree.root()), token=str(token), amount=str(amount), label=label,
        recipient=str(recipient), spend_key=str(spend_key), blinding=str(blinding), siblings=[str(x) for x in sibs],
        path_bits=path_bits, r=str(r), s=str(s), public=[str(x) for x in w[1:7]], proof=proof.hex(),
        vk=dict(alpha1=vkb["alpha1"].hex(), beta2=vkb["beta2"].hex(), gamma2=vkb["gamma2"].hex(), delta2=vkb["delta2"].hex(),
                ic=vkb["ic"].hex()),
        pk_queries_sha256=hashlib.sha256(pkb["a"] + pkb["b1"] + pkb["b2"] + pkb["l"] + pkb["h"]).hexdigest(),
        witness_sha256=hashlib.sha256(wit).hexdigest())
    with open(os.path.join(HERE, "ragequit_vectors.json"), "w") as f:
        json.dump(out, f, indent=1)
    print("wrote ragequit_vectors.json")


if __name__ == "__main__":
    main()
