"""Generates tests/golden/owned_labeled_vectors.json from the spec (oracle/owned_labeled_circuit.py, oracle/groth16.py's setup
exponents) and the oracle's C port (fixed-base multiplications, prover) with a fixed seed: one depth-2 owned labeled transfer
proof with every value injected, its verifying key and the hashes of its proving-key queries and witness.
Run from the repo root after building the oracle (make -C oracle/cpu):  python -m tests.golden.gen_owned_labeled_golden
"""
import hashlib
import json
import os
import random

from oracle import bn254 as bn
from oracle import cport, mimc7
from oracle.labeled_association_circuit import ApprovedTree
from oracle.owned_labeled_circuit import build_r1cs, note_leaf, spend_public_key, witness

R = bn.R
HERE = os.path.dirname(os.path.abspath(__file__))
DEPTH = 2


def main():
    rng = random.Random(20261018)
    cs = build_r1cs(DEPTH)
    tox = [rng.randrange(1, R) for _ in range(5)]
    pkb, vkb = cport.setup_bytes(cs, *tox)
    token, recipient = rng.randrange(1 << 160), rng.randrange(1 << 160)
    tree = mimc7.MerkleTree(DEPTH)
    tree.insert(rng.randrange(R))
    label = 1                                   # the pool index of the deposit both inputs descend from
    notes = [(rng.randrange(R), rng.randrange(R), rng.randrange(1 << 63)) for _ in range(2)]
    idx = [tree.insert(note_leaf(spend_public_key(s), b, token, a, label)) for s, b, a in notes]
    ins = []
    for (s, b, a), i in zip(notes, idx):
        sibs, bits = tree.path(i)
        ins.append((s, b, a, sibs, sum(x << l for l, x in enumerate(bits))))
    withdrawn = rng.randrange(notes[0][2])
    rest = notes[0][2] + notes[1][2] - withdrawn
    out0 = rng.randrange(rest)
    outs = [(spend_public_key(rng.randrange(R)), rng.randrange(R), out0), (spend_public_key(rng.randrange(R)), rng.randrange(R), rest - out0)]
    approved = ApprovedTree(DEPTH, [0, label])
    asibs, abits = approved.path(label)
    abits = sum(x << l for l, x in enumerate(abits))
    r, s = rng.randrange(R), rng.randrange(R)
    w = witness(tree.root(), token, withdrawn, recipient, label, ins, outs, asibs, abits)
    assert cs.is_satisfied(w)
    wit = cport.frs(w)
    proof = cport.Prover(cs, pkb).prove(wit, r, s)
    out = dict(
        depth=DEPTH, toxic=[str(x) for x in tox], root=str(tree.root()), token=str(token), withdrawn=str(withdrawn),
        recipient=str(recipient), label=label,
        inputs=[dict(spend_key=str(k), blinding=str(b), amount=str(a), siblings=[str(x) for x in sb], path_bits=pb)
                for k, b, a, sb, pb in ins],
        outputs=[dict(owner=str(o), blinding=str(b), amount=str(a)) for o, b, a in outs],
        assoc_siblings=[str(x) for x in asibs], assoc_path_bits=abits,
        r=str(r), s=str(s), public=[str(x) for x in w[1:10]], proof=proof.hex(),
        vk=dict(alpha1=vkb["alpha1"].hex(), beta2=vkb["beta2"].hex(), gamma2=vkb["gamma2"].hex(), delta2=vkb["delta2"].hex(),
                ic=vkb["ic"].hex()),
        pk_queries_sha256=hashlib.sha256(pkb["a"] + pkb["b1"] + pkb["b2"] + pkb["l"] + pkb["h"]).hexdigest(),
        witness_sha256=hashlib.sha256(wit).hexdigest())
    with open(os.path.join(HERE, "owned_labeled_vectors.json"), "w") as f:
        json.dump(out, f, indent=1)
    print("wrote owned_labeled_vectors.json")


if __name__ == "__main__":
    main()
