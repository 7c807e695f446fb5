"""The frozen privacy-pool *transfer* statement (two notes in, two notes out, a public amount) as an R1CS, plus its
witness map.

The third statement of the library (DESIGN.md section 3); the product's C++ builder
(owshen_b200/csrc/withdraw_circuit.hpp: TransferBuilder) must reproduce it entry for entry.

A note is (nullifier, secret, token, amount) with amount < 2^64:
  commitment     = MultiMiMC7([nullifier, secret, token, amount], key=0)
  nullifier_hash = MultiMiMC7([nullifier], key=1)          (the withdraw statement's, so a node keeps one nullifier set)

Statement (public: root, public_amount, token, recipient, nullifier_hash[2], out_commitment[2]):
  I know two input notes and two output notes of `token` such that
    nullifier_hash[i]  is input i's nullifier hash, and the two differ;
    every nonzero-valued input note's commitment reaches `root` along its Merkle path;
    out_commitment[j]  is output j's commitment;
    in_amount0 + in_amount1 + public_amount = out_amount0 + out_amount1  (mod r), every amount range-checked to 64 bits;
  and recipient is bound by recipient^2 = recipient_sq.
public_amount below 2^65 is a deposit of that much; above r - 2^65 it is a withdrawal of r - public_amount to recipient.

Variable layout (index -> meaning), P = 4*n_rounds:
  0 ONE
  1 root | 2 public_amount | 3 token | 4 recipient | 5 nh[0] | 6 nh[1] | 7 out_cm[0] | 8 out_cm[1]     (public, n_pub = 8)
  9 recipient_sq | 10 nh_diff_inv
  11..  input block 0, input block 1; each 68 + 5P + depth*(2P + 4) variables:
        +0 nullifier | +1 secret | +2 amount | +3..+66 amount bits, LSB first
        +67 nullifier-hash permutation (P)
        +67+P commitment: 4 permutations (4P), then cm_out
        +68+5P depth levels, each the withdraw statement's level block (sibling, bit, left, perm1[P], perm2[P], out)
  then  output block 0, output block 1; each 68 + 4P variables:
        +0 nullifier | +1 secret | +2 amount | +3..+66 amount bits | +67 commitment (4P) | +67+4P cm_out
Constraint order:
  recipient^2;
  per input: nullifier-hash permutation, (ONE + nullifier + h) * ONE = nh[i]; 64 rows bit*(bit - ONE) = 0,
             (sum 2^k bit_k - amount) * ONE = 0; the commitment's four permutations, r4 * ONE = cm_out;
             the depth levels exactly as withdraw; (root - node_depth) * amount = 0;
  per output: the 65 range rows, the commitment's four permutations and its cm_out row, (cm_out - out_cm[j]) * ONE = 0;
  (in_amount0 + in_amount1 + public_amount - out_amount0 - out_amount1) * ONE = 0;
  (nh[0] - nh[1]) * nh_diff_inv = ONE.
Sizes: n_vars = 283 + 18P + depth*(4P + 8), n_constraints = 273 + 18P + depth*(4P + 6);
with 91 rounds at depth 32 that is 53 683 variables and 53 609 constraints, domain 2^16.
"""
from .bn254 import R
from .mimc7 import N_ROUNDS
from .withdraw_circuit import R1CS, _hash2_witness, _perm_constraints, _perm_witness, lc_add

N_PUB = 8
AMOUNT_BITS = 64
V_ONE, V_ROOT, V_PUB_AMOUNT, V_TOKEN, V_RECIP = range(5)
V_NH = (5, 6)
V_OUT_CM = (7, 8)
V_RSQ, V_NH_INV = 9, 10
V_IN_BASE = 11


class Layout:
    def __init__(self, depth: int, n_rounds: int = N_ROUNDS):
        self.depth, self.n_rounds = depth, n_rounds
        P = self.perm = 4 * n_rounds
        self.lvl_size = 2 * P + 4
        self.in_size = 68 + 5 * P + depth * self.lvl_size
        self.out_size = 68 + 4 * P
        self.out_base = V_IN_BASE + 2 * self.in_size
        self.n_vars = self.out_base + 2 * self.out_size
        self.n_constraints = 273 + 18 * P + depth * (4 * P + 6)
        assert self.n_vars == 283 + 18 * P + depth * (4 * P + 8)

    def note(self, base):
        """Variables of the note block at `base` (input or output): the parts both kinds share."""
        return dict(null=base, sec=base + 1, amount=base + 2, bits=base + 3)

    def inp(self, i):
        b = V_IN_BASE + i * self.in_size
        P = self.perm
        v = self.note(b)
        v.update(nh_perm=b + 67, cm=b + 67 + P, cm_out=b + 67 + 5 * P, lvl_base=b + 68 + 5 * P)
        return v

    def out(self, j):
        b = self.out_base + j * self.out_size
        v = self.note(b)
        v.update(cm=b + 67, cm_out=b + 67 + 4 * self.perm)
        return v

    def level(self, i, l):
        b = self.inp(i)["lvl_base"] + l * self.lvl_size
        P = self.perm
        return dict(sib=b, bit=b + 1, left=b + 2, perm1=b + 3, perm2=b + 3 + P, out=b + 3 + 2 * P)


def _multi_hash_constraints(cs, xs, key_lc, bases, n_rounds):
    """MultiMiMC7(xs, key) over LCs: r = key; r = r + x + hash(x, r) per input, the i-th permutation's rounds at bases[i].
    Returns the LC of the result (the caller binds it to a variable)."""
    r = key_lc
    for x, base in zip(xs, bases):
        h = _perm_constraints(cs, x, r, base, n_rounds)
        r = lc_add(r, x, h)
    return r


def _range_constraints(cs, v):
    for k in range(AMOUNT_BITS):
        b = v["bits"] + k
        cs.add({b: 1}, {b: 1, V_ONE: R - 1}, {})
    packed = {v["bits"] + k: pow(2, k, R) for k in range(AMOUNT_BITS)}
    cs.add(lc_add(packed, {v["amount"]: R - 1}), {V_ONE: 1}, {})


def _commitment_constraints(cs, v, P, n_rounds):
    xs = [{v["null"]: 1}, {v["sec"]: 1}, {V_TOKEN: 1}, {v["amount"]: 1}]
    r4 = _multi_hash_constraints(cs, xs, {}, [v["cm"] + k * P for k in range(4)], n_rounds)
    cs.add(r4, {V_ONE: 1}, {v["cm_out"]: 1})


def build_r1cs(depth: int, n_rounds: int = N_ROUNDS) -> R1CS:
    assert 1 <= depth <= 32
    L = Layout(depth, n_rounds)
    P = L.perm
    cs = R1CS(L.n_vars, N_PUB)
    cs.add({V_RECIP: 1}, {V_RECIP: 1}, {V_RSQ: 1})
    for i in range(2):
        v = L.inp(i)
        nh = _multi_hash_constraints(cs, [{v["null"]: 1}], {V_ONE: 1}, [v["nh_perm"]], n_rounds)
        cs.add(nh, {V_ONE: 1}, {V_NH[i]: 1})
        _range_constraints(cs, v)
        _commitment_constraints(cs, v, P, n_rounds)
        cur = v["cm_out"]
        for l in range(depth):
            lv = L.level(i, l)
            cs.add({lv["bit"]: 1}, lc_add({lv["bit"]: 1}, {V_ONE: R - 1}), {})
            cs.add({lv["bit"]: 1}, lc_add({lv["sib"]: 1}, {cur: R - 1}), lc_add({lv["left"]: 1}, {cur: R - 1}))
            right = lc_add({lv["sib"]: 1}, {cur: 1}, {lv["left"]: R - 1})
            r2 = _multi_hash_constraints(cs, [{lv["left"]: 1}, right], {}, [lv["perm1"], lv["perm2"]], n_rounds)
            cs.add(r2, {V_ONE: 1}, {lv["out"]: 1})
            cur = lv["out"]
        cs.add(lc_add({V_ROOT: 1}, {cur: R - 1}), {v["amount"]: 1}, {})
    for j in range(2):
        v = L.out(j)
        _range_constraints(cs, v)
        _commitment_constraints(cs, v, P, n_rounds)
        cs.add(lc_add({v["cm_out"]: 1}, {V_OUT_CM[j]: R - 1}), {V_ONE: 1}, {})
    i0, i1, o0, o1 = L.inp(0)["amount"], L.inp(1)["amount"], L.out(0)["amount"], L.out(1)["amount"]
    cs.add(lc_add({i0: 1}, {i1: 1}, {V_PUB_AMOUNT: 1}, {o0: R - 1}, {o1: R - 1}), {V_ONE: 1}, {})
    cs.add({V_NH[0]: 1, V_NH[1]: R - 1}, {V_NH_INV: 1}, {V_ONE: 1})
    assert cs.n_constraints == L.n_constraints
    return cs


def _note_witness(w, v, nullifier, secret, token, amount, P, n_rounds):
    """Fills a note block's inputs, the low 64 bits of amount and the commitment; returns the commitment."""
    w[v["null"]], w[v["sec"]], w[v["amount"]] = nullifier % R, secret % R, amount
    for k in range(AMOUNT_BITS):
        w[v["bits"] + k] = (amount >> k) & 1
    r = 0
    for k, x in enumerate((w[v["null"]], w[v["sec"]], token, amount)):
        r = (r + x + _perm_witness(w, x, r, v["cm"] + k * P, n_rounds)) % R
    w[v["cm_out"]] = r
    return r


def witness(root, token, recipient, inputs, outputs, n_rounds: int = N_ROUNDS):
    """Full assignment (list of n_vars ints).
    inputs: two (nullifier, secret, amount, siblings[depth], path_bits) tuples; outputs: two (nullifier, secret, amount).
    root is the caller's; public_amount, the nullifier hashes and the output commitments are derived.  An input of nonzero
    value that does not reach root, or two inputs with one nullifier, give an assignment that does not satisfy the R1CS."""
    depth = len(inputs[0][3])
    assert all(0 <= note[2] < 1 << AMOUNT_BITS for note in list(inputs) + list(outputs)), "amounts are below 2^64"
    L = Layout(depth, n_rounds)
    P = L.perm
    w = [0] * L.n_vars
    w[V_ONE] = 1
    w[V_ROOT] = root % R
    w[V_TOKEN] = token % R
    w[V_RECIP] = recipient % R
    w[V_RSQ] = w[V_RECIP] * w[V_RECIP] % R
    for i, (nul, sec, amount, sibs, bits) in enumerate(inputs):
        assert len(sibs) == depth
        v = L.inp(i)
        nul %= R
        w[V_NH[i]] = (1 + nul + _perm_witness(w, nul, 1, v["nh_perm"], n_rounds)) % R
        cur = _note_witness(w, v, nul, sec, w[V_TOKEN], amount, P, n_rounds)
        for l in range(depth):
            lv = L.level(i, l)
            sib, bit = sibs[l] % R, (bits >> l) & 1
            left, right = (sib, cur) if bit else (cur, sib)
            w[lv["sib"]], w[lv["bit"]], w[lv["left"]] = sib, bit, left
            cur = _hash2_witness(w, left, right, lv["perm1"], lv["perm2"], lv["out"], n_rounds)
    for j, (nul, sec, amount) in enumerate(outputs):
        w[V_OUT_CM[j]] = _note_witness(w, L.out(j), nul, sec, w[V_TOKEN], amount, P, n_rounds)
    a_in = inputs[0][2] + inputs[1][2]
    a_out = outputs[0][2] + outputs[1][2]
    w[V_PUB_AMOUNT] = (a_out - a_in) % R
    d = (w[V_NH[0]] - w[V_NH[1]]) % R
    w[V_NH_INV] = pow(d, R - 2, R) if d else 0
    return w
