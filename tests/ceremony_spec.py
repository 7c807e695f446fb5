"""Two-phase Groth16 setup ceremony, pure Python spec at tiny sizes (DESIGN.md section 4b; Bowe-Gabizon-Miers 2017).

Phase 1 accumulator (M = 2^log_max): [tau^i]_1 (i < 2M), [alpha tau^i]_1, [beta tau^i]_1, [tau^i]_2 (i < M), [beta]_2.
A contribution (t, a, b) multiplies them by t^i, a t^i, b t^i, t^i and b, and publishes [x]_1, [x]_2 and a Schnorr
proof of knowledge for each x.  Key derivation takes the Lagrange bases as inverse NTTs over group elements; the
H query is the odd half of the size-2m basis.  The resulting key equals oracle.groth16.setup(cs, prod t, prod a,
prod b, 1, prod d).
"""
from oracle.bn254 import (R, G1_GEN, G2_GEN, g1_add, g1_mul, g1_neg, g2_add, g2_mul, g1_on_curve, g2_on_curve,
                          g1_msm, g2_msm, g1_to_bytes, g2_to_bytes, g1_from_bytes, g2_from_bytes,
                          root_of_unity)
from oracle.groth16 import domain_log
from oracle.keccak import keccak256
from oracle.pairing import pairing_product_is_one

POK_TAG = b"OG-ceremony-pok"
RHO_TAG = b"OG-ceremony-rho"


def in_g2(q) -> bool:
    """r Q = infinity, written (r-1) Q + Q because g2_mul reduces its scalar mod r"""
    return g2_add(g2_mul(q, R - 1), q) is None


def _le(h: bytes) -> int:
    return int.from_bytes(h, "little") % R


def ptau_new(log_max):
    M = 1 << log_max
    return dict(log_max=log_max, tau1=[G1_GEN] * (2 * M), alpha1=[G1_GEN] * M, beta1=[G1_GEN] * M, tau2=[G2_GEN] * M, beta2=G2_GEN)


def ptau_to_bytes(acc) -> bytes:
    out = b"OGPT" + (1).to_bytes(4, "little") + acc["log_max"].to_bytes(4, "little")
    out += b"".join(g1_to_bytes(p) for p in acc["tau1"] + acc["alpha1"] + acc["beta1"])
    return out + b"".join(g2_to_bytes(p) for p in acc["tau2"] + [acc["beta2"]])


def ptau_from_bytes(b: bytes):
    """None unless the blob has the OGPT v1 layout with log_max in [1, 24] and canonical coordinates."""
    if len(b) < 12 or b[:4] != b"OGPT" or int.from_bytes(b[4:8], "little") != 1:
        return None
    lm = int.from_bytes(b[8:12], "little")
    if not 1 <= lm <= 24 or len(b) != 12 + (384 << lm) + 128:
        return None
    M = 1 << lm
    try:
        g1 = [g1_from_bytes(b[12 + 64 * i:76 + 64 * i]) for i in range(4 * M)]
        o = 12 + 256 * M
        g2 = [g2_from_bytes(b[o + 128 * i:o + 128 * i + 128]) for i in range(M + 1)]
    except ValueError:
        return None
    return dict(log_max=lm, tau1=g1[:2 * M], alpha1=g1[2 * M:3 * M], beta1=g1[3 * M:], tau2=g2[:M], beta2=g2[M])


def pok_challenge(prev_hash, index, x1b, x2b, rb) -> int:
    return _le(keccak256(POK_TAG + prev_hash + index.to_bytes(4, "little") + x1b + x2b + rb))


def make_pok(prev_hash, index, x, k) -> bytes:
    x1b, x2b, rb = g1_to_bytes(g1_mul(G1_GEN, x)), g2_to_bytes(g2_mul(G2_GEN, x)), g1_to_bytes(g1_mul(G1_GEN, k))
    z = (k + pok_challenge(prev_hash, index, x1b, x2b, rb) * x) % R
    return x1b + x2b + rb + z.to_bytes(32, "little")


def check_pok(prev_hash, index, e: bytes):
    """([x]_1, [x]_2) if the entry is a valid proof of knowledge, else None."""
    X1, X2, Rp = g1_from_bytes(e[:64]), g2_from_bytes(e[64:192]), g1_from_bytes(e[192:256])
    z = int.from_bytes(e[256:288], "little")
    if z >= R or None in (X1, X2, Rp) or not (g1_on_curve(X1) and g2_on_curve(X2) and g1_on_curve(Rp)):
        return None
    if not in_g2(X2):
        return None
    c = pok_challenge(prev_hash, index, e[:64], e[64:192], e[192:256])
    if g1_mul(G1_GEN, z) != g1_add(Rp, g1_mul(X1, c)):
        return None
    if not pairing_product_is_one([(X1, G2_GEN), (g1_neg(G1_GEN), X2)]):
        return None
    return X1, X2


def contribute(acc_bytes: bytes, t, a, b, nonces):
    """(new accumulator bytes, OGPR record)"""
    acc = ptau_from_bytes(acc_bytes)
    assert acc is not None and all(x % R for x in (t, a, b, *nonces))
    tp = [pow(t, i, R) for i in range(len(acc["tau1"]))]
    new = dict(log_max=acc["log_max"],
               tau1=[g1_mul(p, s) for p, s in zip(acc["tau1"], tp)],
               alpha1=[g1_mul(p, a * s) for p, s in zip(acc["alpha1"], tp)],
               beta1=[g1_mul(p, b * s) for p, s in zip(acc["beta1"], tp)],
               tau2=[g2_mul(p, s) for p, s in zip(acc["tau2"], tp)],
               beta2=g2_mul(acc["beta2"], b))
    h = keccak256(acc_bytes)
    rec = b"OGPR" + (1).to_bytes(4, "little") + h + b"".join(make_pok(h, i, x, k) for i, (x, k) in enumerate(zip((t, a, b), nonces)))
    return ptau_to_bytes(new), rec


def fs_rho(prev: bytes, nxt: bytes, rec: bytes) -> int:
    return _le(keccak256(RHO_TAG + keccak256(prev) + keccak256(nxt) + keccak256(rec)))


def _pair_eq(p0, q0, p1, q1):
    return pairing_product_is_one([(p0, q0), (g1_neg(p1), q1)])


def ptau_verify(prev: bytes, nxt: bytes, rec: bytes) -> bool:
    A0, A1 = ptau_from_bytes(prev), ptau_from_bytes(nxt)
    if A0 is None or A1 is None or A0["log_max"] != A1["log_max"]:
        return False
    if len(rec) != 904 or rec[:4] != b"OGPR" or int.from_bytes(rec[4:8], "little") != 1 or rec[8:40] != keccak256(prev):
        return False
    X = [check_pok(rec[8:40], i, rec[40 + 288 * i:328 + 288 * i]) for i in range(3)]
    if None in X:
        return False
    g1s = A1["tau1"] + A1["alpha1"] + A1["beta1"]
    g2s = A1["tau2"] + [A1["beta2"]]
    if any(p is None or not g1_on_curve(p) for p in g1s) or any(q is None or not g2_on_curve(q) or not in_g2(q) for q in g2s):
        return False
    if A1["tau1"][0] != G1_GEN or A1["tau2"][0] != G2_GEN:
        return False
    if not (_pair_eq(A1["tau1"][1], G2_GEN, A0["tau1"][1], X[0][1]) and _pair_eq(A1["alpha1"][0], G2_GEN, A0["alpha1"][0], X[1][1])
            and _pair_eq(A1["beta1"][0], G2_GEN, A0["beta1"][0], X[2][1]) and _pair_eq(A1["beta1"][0], G2_GEN, G1_GEN, A1["beta2"])):
        return False
    rho = fs_rho(prev, nxt, rec)
    tau2 = A1["tau2"][1]
    for seq in (A1["tau1"], A1["alpha1"], A1["beta1"]):
        rp = [pow(rho, i, R) for i in range(len(seq) - 1)]
        if not _pair_eq(g1_msm(seq[1:], rp), G2_GEN, g1_msm(seq[:-1], rp), tau2):
            return False
    seq = A1["tau2"]
    rp = [pow(rho, i, R) for i in range(len(seq) - 1)]
    return _pair_eq(G1_GEN, g2_msm(seq[1:], rp), A1["tau1"][1], g2_msm(seq[:-1], rp))


def group_intt(points, add, mul):
    """[(1/m) sum_k omega^-jk P_k]_j, omega = 7^((r-1)/m): the definition, O(m^2)."""
    m = len(points)
    log_m = m.bit_length() - 1
    winv = pow(root_of_unity(log_m), -1, R)
    minv = pow(m, -1, R)
    out = []
    for j in range(m):
        acc = None
        for k, p in enumerate(points):
            acc = add(acc, mul(p, pow(winv, j * k, R) * minv % R))
        out.append(acc)
    return out


def prepare(acc_bytes: bytes, cs):
    """The phase-2 starting key (gamma = delta = 1) as the dicts oracle.groth16.setup returns."""
    acc = ptau_from_bytes(acc_bytes)
    log_m = domain_log(cs.n_constraints, cs.n_pub)
    m = 1 << log_m
    assert log_m <= acc["log_max"]
    L1 = group_intt(acc["tau1"][:m], g1_add, g1_mul)
    aL = group_intt(acc["alpha1"][:m], g1_add, g1_mul)
    bL = group_intt(acc["beta1"][:m], g1_add, g1_mul)
    L2 = group_intt(acc["tau2"][:m], g2_add, g2_mul)
    H = group_intt(acc["tau1"][:2 * m], g1_add, g1_mul)[1::2]
    nv = cs.n_vars
    qa, qb1, qb2, k = [None] * nv, [None] * nv, [None] * nv, [None] * nv
    rows = [(j, cs.A[j], cs.B[j], cs.C[j]) for j in range(cs.n_constraints)]
    rows += [(cs.n_constraints + i, {i: 1}, {}, {}) for i in range(cs.n_pub + 1)]
    for j, Aj, Bj, Cj in rows:
        for i, c in Aj.items():
            qa[i] = g1_add(qa[i], g1_mul(L1[j], c))
            k[i] = g1_add(k[i], g1_mul(bL[j], c))
        for i, c in Bj.items():
            qb1[i] = g1_add(qb1[i], g1_mul(L1[j], c))
            qb2[i] = g2_add(qb2[i], g2_mul(L2[j], c))
            k[i] = g1_add(k[i], g1_mul(aL[j], c))
        for i, c in Cj.items():
            k[i] = g1_add(k[i], g1_mul(L1[j], c))
    pk = dict(log_m=log_m, n_vars=nv, n_pub=cs.n_pub, alpha1=acc["alpha1"][0], beta1=acc["beta1"][0], beta2=acc["beta2"],
              delta1=G1_GEN, delta2=G2_GEN, a=qa, b1=qb1, b2=qb2, l=k[cs.n_pub + 1:], h=H)
    vk = dict(alpha1=pk["alpha1"], beta2=pk["beta2"], gamma2=G2_GEN, delta2=G2_GEN, ic=k[:cs.n_pub + 1])
    return pk, vk


def phase2_contribute(pk, vk, d):
    """delta times d, the L and H queries times 1/d (the record's proof of knowledge is make_pok over the key's hash)."""
    di = pow(d, -1, R)
    pk = dict(pk, delta1=g1_mul(pk["delta1"], d), delta2=g2_mul(pk["delta2"], d),
              l=[g1_mul(p, di) for p in pk["l"]], h=[g1_mul(p, di) for p in pk["h"]])
    return pk, dict(vk, delta2=pk["delta2"])

