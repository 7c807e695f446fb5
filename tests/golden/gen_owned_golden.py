"""Generates tests/golden/owned_vectors.json from the spec (oracle/owned_circuit.py, oracle/groth16.py's setup exponents) and
the oracle's C port (fixed-base multiplications, prover) with a fixed seed: one depth-2 owned transfer proof with every value
injected, its verifying key and the hashes of its proving-key queries and witness.
Run from the repo root after building the oracle (make -C oracle/cpu):  python -m tests.golden.gen_owned_golden
"""
import hashlib
import json
import os
import random

from oracle import bn254 as bn
from oracle import cport, mimc7
from oracle.owned_circuit import build_r1cs, commitment, spend_public_key, witness

R = bn.R
HERE = os.path.dirname(os.path.abspath(__file__))
DEPTH = 2


def main():
    rng = random.Random(20261017)
    cs = build_r1cs(DEPTH)
    tox = [rng.randrange(1, R) for _ in range(5)]
    pkb, vkb = cport.setup_bytes(cs, *tox)
    token, recipient = rng.randrange(1 << 160), rng.randrange(1 << 160)
    tree = mimc7.MerkleTree(DEPTH)
    tree.insert(rng.randrange(R))
    notes = [(rng.randrange(R), rng.randrange(R), rng.randrange(1 << 64)) for _ in range(2)]
    idx = [tree.insert(commitment(spend_public_key(s), b, token, a)) for s, b, a in notes]
    ins = []
    for (s, b, a), i in zip(notes, idx):
        sibs, bits = tree.path(i)
        ins.append((s, b, a, sibs, sum(x << l for l, x in enumerate(bits))))
    outs = [(spend_public_key(rng.randrange(R)), rng.randrange(R), rng.randrange(1 << 64)) for _ in range(2)]
    r, s = rng.randrange(R), rng.randrange(R)
    w = witness(tree.root(), token, recipient, ins, outs)
    assert cs.is_satisfied(w)
    wit = cport.frs(w)
    proof = cport.Prover(cs, pkb).prove(wit, r, s)
    out = dict(
        depth=DEPTH, toxic=[str(x) for x in tox], root=str(tree.root()), token=str(token), recipient=str(recipient),
        inputs=[dict(spend_key=str(k), blinding=str(b), amount=str(a), siblings=[str(x) for x in sb], path_bits=pb)
                for k, b, a, sb, pb in ins],
        outputs=[dict(owner=str(o), blinding=str(b), amount=str(a)) for o, b, a in outs],
        r=str(r), s=str(s), public=[str(x) for x in w[1:9]], proof=proof.hex(),
        vk=dict(alpha1=vkb["alpha1"].hex(), beta2=vkb["beta2"].hex(), gamma2=vkb["gamma2"].hex(), delta2=vkb["delta2"].hex(),
                ic=vkb["ic"].hex()),
        pk_queries_sha256=hashlib.sha256(pkb["a"] + pkb["b1"] + pkb["b2"] + pkb["l"] + pkb["h"]).hexdigest(),
        witness_sha256=hashlib.sha256(wit).hexdigest())
    with open(os.path.join(HERE, "owned_vectors.json"), "w") as f:
        json.dump(out, f, indent=1)
    print("wrote owned_vectors.json")


if __name__ == "__main__":
    main()
