"""Generates tests/golden/labeled_association_vectors.json from the spec (oracle/labeled_association_circuit.py,
oracle/groth16.py's setup exponents) and the oracle's C port (fixed-base multiplications, prover) with a fixed seed: one
depth-2 labeled association withdraw proof (a partial withdrawal with change) with every value injected, its verifying key
and the hashes of its proving-key queries and witness.
Run from the repo root after building the oracle (make -C oracle/cpu):  python -m tests.golden.gen_labeled_association_golden
"""
import hashlib
import json
import os
import random

from oracle import bn254 as bn
from oracle import cport, mimc7
from oracle.labeled_association_circuit import ApprovedTree, build_r1cs, leaf, precommitment, witness

R = bn.R
HERE = os.path.dirname(os.path.abspath(__file__))
DEPTH = 2


def main():
    rng = random.Random(20261017)
    cs = build_r1cs(DEPTH)
    tox = [rng.randrange(1, R) for _ in range(5)]
    pkb, vkb = cport.setup_bytes(cs, *tox)
    nullifier, secret, recipient, token = rng.randrange(R), rng.randrange(R), rng.randrange(1 << 160), rng.randrange(R)
    amount = rng.randrange(1 << 64)
    withdrawn = rng.randrange(amount)
    change_nullifier, change_secret = rng.randrange(R), rng.randrange(R)
    pool = mimc7.MerkleTree(DEPTH)
    pool.insert(rng.randrange(R))
    label = pool.n_leaves                                # the deposit's index; the provider approves it after deposit 3
    i = pool.insert(leaf(precommitment(nullifier, secret), token, amount, label))
    pool.insert(rng.randrange(R))
    approved = ApprovedTree(DEPTH, [3, label])
    sibs, bits = pool.path(i)
    asibs, abits = approved.path(label)
    r, s = rng.randrange(R), rng.randrange(R)
    w = witness(nullifier, secret, recipient, token, withdrawn, amount, label, sibs, bits, change_nullifier, change_secret, asibs, abits)
    assert cs.is_satisfied(w) and (w[1], w[4]) == (pool.root(), approved.root())
    assert w[7] == leaf(precommitment(change_nullifier, change_secret), token, amount - withdrawn, label)
    wit = cport.frs(w)
    proof = cport.Prover(cs, pkb).prove(wit, r, s)
    pack = lambda bs: sum(b << l for l, b in enumerate(bs))
    out = dict(
        depth=DEPTH, toxic=[str(x) for x in tox], token=str(token), recipient=str(recipient), withdrawn=withdrawn,
        nullifier=str(nullifier), secret=str(secret), amount=amount, label=label, siblings=[str(x) for x in sibs],
        path_bits=pack(bits), change_nullifier=str(change_nullifier), change_secret=str(change_secret), approved=approved.labels,
        assoc_siblings=[str(x) for x in asibs], assoc_path_bits=pack(abits),
        r=str(r), s=str(s), public=[str(x) for x in w[1:8]], proof=proof.hex(),
        vk=dict(alpha1=vkb["alpha1"].hex(), beta2=vkb["beta2"].hex(), gamma2=vkb["gamma2"].hex(), delta2=vkb["delta2"].hex(),
                ic=vkb["ic"].hex()),
        pk_queries_sha256=hashlib.sha256(pkb["a"] + pkb["b1"] + pkb["b2"] + pkb["l"] + pkb["h"]).hexdigest(),
        witness_sha256=hashlib.sha256(wit).hexdigest())
    with open(os.path.join(HERE, "labeled_association_vectors.json"), "w") as f:
        json.dump(out, f, indent=1)
    print("wrote labeled_association_vectors.json")


if __name__ == "__main__":
    main()
