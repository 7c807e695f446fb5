"""Generates tests/golden/deposit_vectors.json from the pure-Python spec (oracle/deposit_circuit.py, oracle/groth16.py)
with a fixed seed: one deposit proof with every value injected, its verifying key and the hashes of its proving-key
queries and witness.
Run from the repo root:  python -m tests.golden.gen_deposit_golden      (~2 minutes, pure Python Groth16)
"""
import hashlib
import json
import os
import random

from oracle import bn254 as bn
from oracle import groth16 as g16
from oracle import mimc7
from oracle.deposit_circuit import build_r1cs, witness

R = bn.R
HERE = os.path.dirname(os.path.abspath(__file__))


def main():
    rng = random.Random(20261015)
    cs = build_r1cs()
    tox = [rng.randrange(1, R) for _ in range(5)]
    pk, vk = g16.setup(cs, *tox)
    nul, sec, dep, r, s = (rng.randrange(R) for _ in range(5))
    w = witness(nul, sec, dep)
    assert cs.is_satisfied(w) and w[1] == mimc7.multi_hash([nul, sec])
    proof = g16.prove(cs, pk, w, r, s)
    assert g16.verify(vk, w[1:3], proof)
    pk_bytes = (b"".join(map(bn.g1_to_bytes, pk["a"])) + b"".join(map(bn.g1_to_bytes, pk["b1"])) + b"".join(map(bn.g2_to_bytes, pk["b2"]))
                + b"".join(map(bn.g1_to_bytes, pk["l"])) + b"".join(map(bn.g1_to_bytes, pk["h"])))
    out = dict(
        toxic=[str(x) for x in tox], nullifier=str(nul), secret=str(sec), depositor=str(dep), r=str(r), s=str(s),
        public=[str(x) for x in w[1:3]], proof=g16.proof_to_bytes(proof).hex(),
        vk=dict(alpha1=bn.g1_to_bytes(vk["alpha1"]).hex(), beta2=bn.g2_to_bytes(vk["beta2"]).hex(),
                gamma2=bn.g2_to_bytes(vk["gamma2"]).hex(), delta2=bn.g2_to_bytes(vk["delta2"]).hex(),
                ic=b"".join(map(bn.g1_to_bytes, vk["ic"])).hex()),
        pk_queries_sha256=hashlib.sha256(pk_bytes).hexdigest(),
        witness_sha256=hashlib.sha256(b"".join(map(bn.fr_to_bytes, w))).hexdigest())
    with open(os.path.join(HERE, "deposit_vectors.json"), "w") as f:
        json.dump(out, f, indent=1)
    print("wrote deposit_vectors.json")


if __name__ == "__main__":
    main()
