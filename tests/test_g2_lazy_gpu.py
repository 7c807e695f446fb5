"""The G2 bucket accumulation (lazily reduced Fq2, ec.cuh: g2_madd_lazy) driven through buckets that meet P + P and P - P on
purpose: a one-shot G2 MSM whose table repeats points and their negations under the same scalar, so that in every window the
copies land in the same bucket.  Compared with the oracle's fixed-base multiplication and its CPU MSM on the same bytes."""
import random

import pytest

import owshen_b200 as ob
from oracle import bn254 as bn
from oracle import cport

R, P = bn.R, bn.P
GEN = bn.g2_to_bytes(bn.G2_GEN)


def _neg(pt):
    y0, y1 = int.from_bytes(pt[64:96], "little"), int.from_bytes(pt[96:], "little")
    return pt[:64] + ((P - y0) % P).to_bytes(32, "little") + ((P - y1) % P).to_bytes(32, "little")


@pytest.mark.gpu
@pytest.mark.parametrize("n_distinct", [256, 1024])
def test_g2_msm_buckets_meet_doubling_and_cancellation(n_distinct):
    rng = random.Random(77 + n_distinct)
    ctx = ob.Context(0)
    d = [rng.randrange(1, R) for _ in range(n_distinct)]
    base = ctx.g2_generator_mul(cport.frs(d))
    pts, logs, ks = [], [], []
    for i in range(n_distinct):
        p, k = base[128 * i:128 * i + 128], rng.randrange(1, R)
        # copies under the same scalar share every bucket: P + P (doubling), then P - P (back to the previous sum or to
        # infinity), three copies and a negation, and once in a while infinity in between
        pattern = [(p, d[i]), (p, d[i])] if i % 4 == 0 else \
                  [(p, d[i]), (_neg(p), R - d[i])] if i % 4 == 1 else \
                  [(p, d[i]), (p, d[i]), (p, d[i]), (_neg(p), R - d[i])] if i % 4 == 2 else \
                  [(p, d[i]), (bytes(128), 0), (p, d[i])]
        for q, lq in pattern:
            pts.append(q); logs.append(lq); ks.append(k)
    order = list(range(len(pts)))
    rng.shuffle(order)
    pts = b"".join(pts[j] for j in order)
    logs = [logs[j] for j in order]
    ks = [ks[j] for j in order]
    t = sum(a * b for a, b in zip(logs, ks)) % R
    exp = cport.g2_fixed_mul_batch(GEN, cport.frs([t]))
    assert cport.g2_msm(pts, cport.frs(ks)) == exp
    assert ctx.msm_g2(pts, cport.frs(ks)) == exp
    ctx.close()
