"""Writes tests/golden/ceremony_vectors.json: a log_max = 2 powers-of-tau ceremony with two fixed contributors, from the
pure-Python spec (tests/ceremony_spec.py) -- every accumulator (hex) and every phase-1 record (hex).
Usage: python -m tests.golden.gen_ceremony_golden"""
import json
import os

from tests import ceremony_spec as spec

CONTRIBUTORS = [dict(secrets=[3, 5, 7], nonces=[11, 13, 17]),
                dict(secrets=[2 ** 200 + 19, 2 ** 100 + 23, 29], nonces=[31, 2 ** 250 + 37, 41])]


def main():
    acc = spec.ptau_to_bytes(spec.ptau_new(2))
    accs, recs = [acc.hex()], []
    for c in CONTRIBUTORS:
        acc, rec = spec.contribute(acc, *c["secrets"], c["nonces"])
        accs.append(acc.hex()); recs.append(rec.hex())
    out = os.path.join(os.path.dirname(os.path.abspath(__file__)), "ceremony_vectors.json")
    json.dump(dict(log_max=2, contributors=CONTRIBUTORS, accumulators=accs, records=recs), open(out, "w"), indent=1)
    print("wrote", out)


if __name__ == "__main__":
    main()
