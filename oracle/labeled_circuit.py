"""The frozen privacy-pool *labeled withdraw* statement as an R1CS, plus its witness map and the labeled note format.

The sixth statement of the library (DESIGN.md section 3); the product's C++ builder
(owshen_b200/csrc/withdraw_circuit.hpp: LabeledBuilder) must reproduce it entry for entry.  A labeled note carries a value and
the identity of the deposit it descends from, its label, so that a compliance provider's blocklist of deposits follows the
value through partial withdrawals (the note of Buterin, Illum, Nadler, Schaer and Soleimani, "Blockchain Privacy and
Regulatory Compliance: Towards a Practical Equilibrium", 2023, and of the Privacy Pools protocol deployed since then).

A labeled note is (nullifier, secret, token, amount < 2^64, label < 2^32):
  precommitment  = MultiMiMC7([nullifier, secret], key=2)
  leaf           = MultiMiMC7([precommitment, token, amount, label], key=2)
  nullifier_hash = MultiMiMC7([nullifier], key=1)          (every statement's, so a node keeps one nullifier set)
Key 2 is the domain separation: MultiMiMC7([pre, token, amount, label], 0) would be a transfer note commitment with
nullifier = pre, secret = token, token = amount and amount = label, all public at deposit.  Key 0 is taken by commitments and
Merkle nodes, key 1 by nullifier hashes.
The label is the pool leaf index at which the node appended the deposit: the depositor sends (precommitment, token, amount)
and the node computes the leaf from them and the index it assigns.  So a blocklist of deposit indices (the exclusion
statement's tree, oracle/exclusion_circuit.py) applies to labeled notes unchanged.

Statement (public: root, nullifier_hash, recipient, exclusion_root, token, withdrawn, change_commitment):
  I know (nullifier, secret, amount, label, siblings[depth], bits[depth], change_nullifier, change_secret, low, next,
          excl_siblings[depth], excl_bits[depth]) such that
    nullifier_hash is the note's nullifier hash;
    the note's leaf (with the public token) reaches root along (siblings, bits);
    amount, withdrawn and change = amount - withdrawn are below 2^64, label is below 2^32;
    change_commitment = MultiMiMC7([MultiMiMC7([change_nullifier, change_secret], 2), token, change, label], 2);
    with x = label + 1: low, next, x - low - 1 and next - x - 1 are below 2^33, and MultiMiMC7([low, next], 0) reaches
    exclusion_root along (excl_siblings, excl_bits);
  and recipient is bound by recipient^2 = recipient_sq.
The range check on withdrawn stops withdrawn = r - k (change = amount + k would mint k); the one on change is
withdrawn <= amount.  change 0 (a full withdrawal) and withdrawn 0 (the note replaced) are both valid.

Variable layout (index -> meaning), P = 4*n_rounds, a level block is the withdraw statement's 2P + 4 variables:
  0 ONE | 1 root | 2 nullifier_hash | 3 recipient | 4 exclusion_root | 5 token | 6 withdrawn | 7 change_commitment
                                                                                                  (public, n_pub = 7)
  8 nullifier | 9 secret | 10 recipient_sq | 11 amount | 12 label | 13 change_nullifier | 14 change_secret | 15 low | 16 next
  17 .. 17+P                       nullifier-hash permutation
  then precommitment block         perm1[P] perm2[P] out
  then leaf block                  perm[4P] out
  then depth pool levels
  then amount bits[64] | withdrawn bits[64] | change bits[64] | label bits[32] | low, next, gap_lo, gap_hi bits[33 each]
                                                                                                  (LSB first)
  then change precommitment block  perm1[P] perm2[P] out
  then change commitment block     perm[4P]        (its output is change_commitment itself)
  then blocklist leaf block        perm1[P] perm2[P] out
  then depth exclusion levels
Constraint order: recipient; nullifier-hash perm rounds, its output; precommitment perm1, perm2, output; leaf perm[4], output;
per pool level: boolean, select, perm1, perm2, output; (cur - root) * ONE = 0; the eight range checks in the order of the
bits above (n rows bit * (bit - ONE) = 0, then (sum 2^k bit_k - value) * ONE = 0); change precommitment perm1, perm2,
output; change commitment perm[4], output r4 * ONE = change_commitment; blocklist leaf perm1, perm2, output; the exclusion
levels, then (cur - exclusion_root) * ONE = 0.
Sizes: n_vars = 377 + 15P + depth*(4P + 8), n_constraints = 373 + 15P + depth*(4P + 6); with 91 rounds at depth 32 that is
52 685 variables and 52 617 constraints, domain 2^16.
"""
from .bn254 import R
from .mimc7 import N_ROUNDS, multi_hash
from .withdraw_circuit import R1CS, _hash2_constraints, _hash2_witness, _perm_constraints, _perm_witness, lc_add, lc_scale

N_PUB = 7
KEY = 2
AMOUNT_BITS, LABEL_BITS, KEY_BITS = 64, 32, 33
(V_ONE, V_ROOT, V_NHASH, V_RECIP, V_XROOT, V_TOKEN, V_WITHDRAWN, V_CHANGE_CM, V_NULL, V_SECRET, V_RSQ, V_AMOUNT, V_LABEL,
 V_CNULL, V_CSECRET, V_LOW, V_NEXT) = range(17)
V_NH_PERM = 17
POOL, EXCL = 0, 1
AMOUNT, WITHDRAWN, CHANGE, LABEL, LOW, NEXT, GAP_LO, GAP_HI = range(8)
RANGE_WIDTHS = (AMOUNT_BITS, AMOUNT_BITS, AMOUNT_BITS, LABEL_BITS, KEY_BITS, KEY_BITS, KEY_BITS, KEY_BITS)


def precommitment(nullifier, secret, n_rounds: int = N_ROUNDS) -> int:
    return multi_hash([nullifier % R, secret % R], KEY, n_rounds)


def leaf(pre, token, amount, label, n_rounds: int = N_ROUNDS) -> int:
    return multi_hash([pre % R, token % R, amount % R, label % R], KEY, n_rounds)


class Layout:
    def __init__(self, depth: int, n_rounds: int = N_ROUNDS):
        self.depth, self.n_rounds = depth, n_rounds
        P = self.perm = 4 * n_rounds
        self.lvl_size = 2 * P + 4
        self.pre_base = V_NH_PERM + P
        self.pre_out = self.pre_base + 2 * P
        self.leaf_base = self.pre_out + 1
        self.leaf_out = self.leaf_base + 4 * P
        self.pool_base = self.leaf_out + 1
        self.bits_base = self.pool_base + depth * self.lvl_size
        self.cpre_base = self.bits_base + sum(RANGE_WIDTHS)
        self.cpre_out = self.cpre_base + 2 * P
        self.ccm_base = self.cpre_out + 1
        self.xleaf_base = self.ccm_base + 4 * P
        self.xleaf_out = self.xleaf_base + 2 * P
        self.excl_base = self.xleaf_out + 1
        self.tree_base = (self.pool_base, self.excl_base)
        self.n_vars = self.excl_base + depth * self.lvl_size
        self.n_constraints = 373 + 15 * P + depth * (4 * P + 6)
        assert self.n_vars == 377 + 15 * P + depth * (4 * P + 8)
        if n_rounds == N_ROUNDS:
            assert (self.n_vars, self.n_constraints) == (5837 + 1464 * depth, 5833 + 1462 * depth)
        # named rows, for the soundness tests
        self.row_pool_root = 7 * P + 4 + depth * (2 * P + 3)
        self.row_range = self.row_pool_root + 1
        self.row_change_cm = self.row_range + sum(w + 1 for w in RANGE_WIDTHS) + 6 * P + 1
        self.row_excl_root = self.n_constraints - 1

    def level(self, tree, l):
        b = self.tree_base[tree] + l * self.lvl_size
        P = self.perm
        return dict(sib=b, bit=b + 1, left=b + 2, perm1=b + 3, perm2=b + 3 + P, out=b + 3 + 2 * P)

    def bits(self, block):
        """First variable of range block AMOUNT, WITHDRAWN, CHANGE, LABEL, LOW, NEXT, GAP_LO or GAP_HI."""
        return self.bits_base + sum(RANGE_WIDTHS[:block])

    def packed_row(self, block):
        """Row (sum 2^k bit_k - value) * ONE = 0 of a range block."""
        return self.row_range + sum(w + 1 for w in RANGE_WIDTHS[:block]) + RANGE_WIDTHS[block]


def _multi_hash_constraints(cs, xs, key_lc, bases, n_rounds):
    r = key_lc
    for x, base in zip(xs, bases):
        h = _perm_constraints(cs, x, r, base, n_rounds)
        r = lc_add(r, x, h)
    return r


def _range_constraints(cs, value, bits, n_bits):
    for k in range(n_bits):
        cs.add({bits + k: 1}, {bits + k: 1, V_ONE: R - 1}, {})
    packed = {bits + k: pow(2, k, R) for k in range(n_bits)}
    cs.add(lc_add(packed, lc_scale(value, R - 1)), {V_ONE: 1}, {})


def _merkle_constraints(cs, L, tree, cur, root):
    for l in range(L.depth):
        v = L.level(tree, l)
        cs.add({v["bit"]: 1}, lc_add({v["bit"]: 1}, {V_ONE: R - 1}), {})
        cs.add({v["bit"]: 1}, lc_add({v["sib"]: 1}, {cur: R - 1}), lc_add({v["left"]: 1}, {cur: R - 1}))
        right = lc_add({v["sib"]: 1}, {cur: 1}, {v["left"]: R - 1})
        _hash2_constraints(cs, {v["left"]: 1}, right, v["perm1"], v["perm2"], v["out"], L.n_rounds)
        cur = v["out"]
    cs.add(lc_add({cur: 1}, {root: R - 1}), {V_ONE: 1}, {})


def build_r1cs(depth: int, n_rounds: int = N_ROUNDS) -> R1CS:
    assert 1 <= depth <= 32
    L = Layout(depth, n_rounds)
    P = L.perm
    cs = R1CS(L.n_vars, N_PUB)
    key = {V_ONE: KEY}
    cs.add({V_RECIP: 1}, {V_RECIP: 1}, {V_RSQ: 1})
    nh = _multi_hash_constraints(cs, [{V_NULL: 1}], {V_ONE: 1}, [V_NH_PERM], n_rounds)
    cs.add(nh, {V_ONE: 1}, {V_NHASH: 1})
    pre = _multi_hash_constraints(cs, [{V_NULL: 1}, {V_SECRET: 1}], key, [L.pre_base, L.pre_base + P], n_rounds)
    cs.add(pre, {V_ONE: 1}, {L.pre_out: 1})
    xs = [{L.pre_out: 1}, {V_TOKEN: 1}, {V_AMOUNT: 1}, {V_LABEL: 1}]
    lf = _multi_hash_constraints(cs, xs, key, [L.leaf_base + k * P for k in range(4)], n_rounds)
    cs.add(lf, {V_ONE: 1}, {L.leaf_out: 1})
    _merkle_constraints(cs, L, POOL, L.leaf_out, V_ROOT)
    change = {V_AMOUNT: 1, V_WITHDRAWN: R - 1}
    x = {V_LABEL: 1, V_ONE: 1}
    values = ({V_AMOUNT: 1}, {V_WITHDRAWN: 1}, change, {V_LABEL: 1}, {V_LOW: 1}, {V_NEXT: 1},
              lc_add(x, {V_LOW: R - 1}, {V_ONE: R - 1}), lc_add({V_NEXT: 1}, lc_scale(x, R - 1), {V_ONE: R - 1}))
    for block, value in enumerate(values):
        _range_constraints(cs, value, L.bits(block), RANGE_WIDTHS[block])
    cpre = _multi_hash_constraints(cs, [{V_CNULL: 1}, {V_CSECRET: 1}], key, [L.cpre_base, L.cpre_base + P], n_rounds)
    cs.add(cpre, {V_ONE: 1}, {L.cpre_out: 1})
    xs = [{L.cpre_out: 1}, {V_TOKEN: 1}, change, {V_LABEL: 1}]
    ccm = _multi_hash_constraints(cs, xs, key, [L.ccm_base + k * P for k in range(4)], n_rounds)
    cs.add(ccm, {V_ONE: 1}, {V_CHANGE_CM: 1})
    _hash2_constraints(cs, {V_LOW: 1}, {V_NEXT: 1}, L.xleaf_base, L.xleaf_base + P, L.xleaf_out, n_rounds)
    _merkle_constraints(cs, L, EXCL, L.xleaf_out, V_XROOT)
    assert cs.n_constraints == L.n_constraints
    return cs


def _multi_hash_witness(w, xs, key, bases, out, n_rounds):
    r = key
    for x, base in zip(xs, bases):
        r = (r + x + _perm_witness(w, x, r, base, n_rounds)) % R
    if out is not None:
        w[out] = r
    return r


def witness(nullifier, secret, recipient, token, withdrawn, amount, label, siblings, bits, change_nullifier, change_secret,
            low, next_, excl_siblings, excl_bits, n_rounds: int = N_ROUNDS):
    """Full assignment (list of n_vars ints).  bits / excl_bits: one bit per level, leaf first.  root, exclusion_root,
    nullifier_hash and change_commitment are derived.  Every range block holds the low bits of the canonical value (mod r)
    it checks, so an overdraw, a withdrawn value of 2^64 or more, a label or amount out of range, a flagged label or a leaf
    that does not bracket it give an assignment that does not satisfy the R1CS."""
    depth = len(siblings)
    assert len(bits) == len(excl_siblings) == len(excl_bits) == depth
    L = Layout(depth, n_rounds)
    P = L.perm
    w = [0] * L.n_vars
    w[V_ONE] = 1
    w[V_RECIP] = recipient % R
    w[V_RSQ] = w[V_RECIP] * w[V_RECIP] % R
    w[V_TOKEN], w[V_WITHDRAWN] = token % R, withdrawn % R
    w[V_NULL], w[V_SECRET], w[V_AMOUNT], w[V_LABEL] = nullifier % R, secret % R, amount % R, label % R
    w[V_CNULL], w[V_CSECRET], w[V_LOW], w[V_NEXT] = change_nullifier % R, change_secret % R, low % R, next_ % R
    w[V_NHASH] = _multi_hash_witness(w, [w[V_NULL]], 1, [V_NH_PERM], None, n_rounds)
    pre = _multi_hash_witness(w, [w[V_NULL], w[V_SECRET]], KEY, [L.pre_base, L.pre_base + P], L.pre_out, n_rounds)
    cur = _multi_hash_witness(w, [pre, w[V_TOKEN], w[V_AMOUNT], w[V_LABEL]], KEY, [L.leaf_base + k * P for k in range(4)],
                              L.leaf_out, n_rounds)
    change = (w[V_AMOUNT] - w[V_WITHDRAWN]) % R
    x = w[V_LABEL] + 1
    values = (w[V_AMOUNT], w[V_WITHDRAWN], change, w[V_LABEL], w[V_LOW], w[V_NEXT], (x - w[V_LOW] - 1) % R,
              (w[V_NEXT] - x - 1) % R)
    for block, value in enumerate(values):
        for k in range(RANGE_WIDTHS[block]):
            w[L.bits(block) + k] = (value >> k) & 1
    cpre = _multi_hash_witness(w, [w[V_CNULL], w[V_CSECRET]], KEY, [L.cpre_base, L.cpre_base + P], L.cpre_out, n_rounds)
    w[V_CHANGE_CM] = _multi_hash_witness(w, [cpre, w[V_TOKEN], change, w[V_LABEL]], KEY, [L.ccm_base + k * P for k in range(4)],
                                         None, n_rounds)
    xleaf = _hash2_witness(w, w[V_LOW], w[V_NEXT], L.xleaf_base, L.xleaf_base + P, L.xleaf_out, n_rounds)
    for tree, root, sibs, bs, cur in ((POOL, V_ROOT, siblings, bits, cur), (EXCL, V_XROOT, excl_siblings, excl_bits, xleaf)):
        for l in range(depth):
            v = L.level(tree, l)
            sib, bit = sibs[l] % R, bs[l] & 1
            left, right = (sib, cur) if bit else (cur, sib)
            w[v["sib"]], w[v["bit"]], w[v["left"]] = sib, bit, left
            cur = _hash2_witness(w, left, right, v["perm1"], v["perm2"], v["out"], n_rounds)
        w[root] = cur
    return w
