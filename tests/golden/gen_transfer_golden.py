"""Generates tests/golden/transfer_vectors.json from the spec (oracle/transfer_circuit.py, oracle/groth16.py's setup
exponents) and the oracle's C port (fixed-base multiplications, prover) with a fixed seed: one depth-2 transfer proof with
every value injected, its verifying key and the hashes of its proving-key queries and witness.
Run from the repo root after building the oracle (make -C oracle/cpu):  python -m tests.golden.gen_transfer_golden
"""
import hashlib
import json
import os
import random

from oracle import bn254 as bn
from oracle import cport, mimc7
from oracle.transfer_circuit import build_r1cs, witness

R = bn.R
HERE = os.path.dirname(os.path.abspath(__file__))
DEPTH = 2


def main():
    rng = random.Random(20261016)
    cs = build_r1cs(DEPTH)
    tox = [rng.randrange(1, R) for _ in range(5)]
    pkb, vkb = cport.setup_bytes(cs, *tox)
    token, recipient = rng.randrange(1 << 160), rng.randrange(1 << 160)
    tree = mimc7.MerkleTree(DEPTH)
    tree.insert(rng.randrange(R))
    notes = [(rng.randrange(R), rng.randrange(R), rng.randrange(1 << 64)) for _ in range(2)]
    idx = [tree.insert(mimc7.multi_hash([n, s, token, a])) for n, s, a in notes]
    ins = []
    for (n, s, a), i in zip(notes, idx):
        sibs, bits = tree.path(i)
        ins.append((n, s, a, sibs, sum(b << l for l, b in enumerate(bits))))
    outs = [(rng.randrange(R), rng.randrange(R), rng.randrange(1 << 64)) for _ in range(2)]
    r, s = rng.randrange(R), rng.randrange(R)
    w = witness(tree.root(), token, recipient, ins, outs)
    assert cs.is_satisfied(w)
    wit = cport.frs(w)
    proof = cport.Prover(cs, pkb).prove(wit, r, s)
    out = dict(
        depth=DEPTH, toxic=[str(x) for x in tox], root=str(tree.root()), token=str(token), recipient=str(recipient),
        inputs=[dict(nullifier=str(n), secret=str(s_), amount=str(a), siblings=[str(x) for x in sb], path_bits=b)
                for n, s_, a, sb, b in ins],
        outputs=[dict(nullifier=str(n), secret=str(s_), amount=str(a)) for n, s_, a in outs],
        r=str(r), s=str(s), public=[str(x) for x in w[1:9]], proof=proof.hex(),
        vk=dict(alpha1=vkb["alpha1"].hex(), beta2=vkb["beta2"].hex(), gamma2=vkb["gamma2"].hex(), delta2=vkb["delta2"].hex(),
                ic=vkb["ic"].hex()),
        pk_queries_sha256=hashlib.sha256(pkb["a"] + pkb["b1"] + pkb["b2"] + pkb["l"] + pkb["h"]).hexdigest(),
        witness_sha256=hashlib.sha256(wit).hexdigest())
    with open(os.path.join(HERE, "transfer_vectors.json"), "w") as f:
        json.dump(out, f, indent=1)
    print("wrote transfer_vectors.json")


if __name__ == "__main__":
    main()
