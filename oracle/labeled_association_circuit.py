"""The frozen privacy-pool *labeled association withdraw* statement as an R1CS, plus its witness map and the provider's tree of
approved labels.

The seventh statement of the library (DESIGN.md section 3); the product's C++ builder
(owshen_b200/csrc/withdraw_circuit.hpp: LabeledAssociationBuilder) must reproduce it entry for entry.  It spends a labeled
note (oracle/labeled_circuit.py) exactly as the labeled statement does, but proves the note's label is on an association set
provider's list of approved deposits (an allow-list) instead of off a blocklist: the model of the Privacy Pools protocol,
where a withdrawal proves its label is in the provider's approved set.

The approved-label tree: a tree of the pool's depth whose leaves are L + 1 for every approved label L (a pool leaf index,
below 2^depth), in any order; every other leaf is 0, as in MerkleTree.  The leaf is not hashed: the set is public anyway,
the fixed path length means only a level-0 value can start a path, and a level-0 value of a published tree is 0 or an
approved L + 1.  The + 1 keeps label 0 (the first deposit) apart from the empty slots, and the 32-bit range check on the
label makes L + 1 nonzero (label = r - 1 would give assoc_leaf = 0, an empty slot).

Statement (public: root, nullifier_hash, recipient, association_root, token, withdrawn, change_commitment):
  I know (nullifier, secret, amount, label, siblings[depth], bits[depth], change_nullifier, change_secret,
          assoc_siblings[depth], assoc_bits[depth]) such that
    the labeled statement's note part holds (nullifier hash, leaf under root, the 64-bit ranges of amount, withdrawn and
    change = amount - withdrawn, the 32-bit range of label, change_commitment);
    assoc_leaf = label + 1, and assoc_leaf reaches association_root along (assoc_siblings, assoc_bits);
  and recipient is bound by recipient^2 = recipient_sq.

Variable layout (index -> meaning), P = 4*n_rounds, a level block is the withdraw statement's 2P + 4 variables:
  0 ONE | 1 root | 2 nullifier_hash | 3 recipient | 4 association_root | 5 token | 6 withdrawn | 7 change_commitment
                                                                                                  (public, n_pub = 7)
  8 nullifier | 9 secret | 10 recipient_sq | 11 amount | 12 label | 13 change_nullifier | 14 change_secret | 15 assoc_leaf
  16 .. 16+P                       nullifier-hash permutation
  then precommitment block         perm1[P] perm2[P] out
  then leaf block                  perm[4P] out
  then depth pool levels
  then amount bits[64] | withdrawn bits[64] | change bits[64] | label bits[32]                   (LSB first)
  then change precommitment block  perm1[P] perm2[P] out
  then change commitment block     perm[4P]        (its output is change_commitment itself)
  then depth association levels
Constraint order: recipient; nullifier-hash perm rounds, its output; precommitment perm1, perm2, output; leaf perm[4], output;
per pool level: boolean, select, perm1, perm2, output; (cur - root) * ONE = 0; the four range checks in the order of the
bits above; change precommitment perm1, perm2, output; change commitment perm[4], output r4 * ONE = change_commitment;
(label + ONE - assoc_leaf) * ONE = 0; the association levels, then (cur - association_root) * ONE = 0.
Sizes: n_vars = 243 + 13P + depth*(4P + 8), n_constraints = 237 + 13P + depth*(4P + 6); with 91 rounds at depth 32 that is
51 823 variables and 51 753 constraints, domain 2^16.
"""
from .bn254 import R
from .labeled_circuit import KEY, _merkle_constraints, _multi_hash_constraints, _multi_hash_witness, _range_constraints, leaf, precommitment
from .mimc7 import N_ROUNDS, MerkleTree
from .withdraw_circuit import R1CS, _hash2_witness, lc_add

N_PUB = 7
AMOUNT_BITS, LABEL_BITS = 64, 32
(V_ONE, V_ROOT, V_NHASH, V_RECIP, V_AROOT, V_TOKEN, V_WITHDRAWN, V_CHANGE_CM, V_NULL, V_SECRET, V_RSQ, V_AMOUNT, V_LABEL,
 V_CNULL, V_CSECRET, V_ALEAF) = range(16)
V_NH_PERM = 16
POOL, ASSOC = 0, 1
AMOUNT, WITHDRAWN, CHANGE, LABEL = range(4)
RANGE_WIDTHS = (AMOUNT_BITS, AMOUNT_BITS, AMOUNT_BITS, LABEL_BITS)


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
        self.assoc_base = self.ccm_base + 4 * P
        self.tree_base = (self.pool_base, self.assoc_base)
        self.n_vars = self.assoc_base + depth * self.lvl_size
        self.n_constraints = 237 + 13 * P + depth * (4 * P + 6)
        assert self.n_vars == 243 + 13 * P + depth * (4 * P + 8)
        if n_rounds == N_ROUNDS:
            assert (self.n_vars, self.n_constraints) == (4975 + 1464 * depth, 4969 + 1462 * depth)
        # named rows, for the soundness tests
        self.row_pool_root = 7 * P + 4 + depth * (2 * P + 3)
        self.row_range = self.row_pool_root + 1
        self.row_change_cm = self.row_range + sum(w + 1 for w in RANGE_WIDTHS) + 6 * P + 1
        self.row_assoc_leaf = self.row_change_cm + 1
        self.row_assoc_root = self.n_constraints - 1

    def level(self, tree, l):
        b = self.tree_base[tree] + l * self.lvl_size
        P = self.perm
        return dict(sib=b, bit=b + 1, left=b + 2, perm1=b + 3, perm2=b + 3 + P, out=b + 3 + 2 * P)

    def bits(self, block):
        """First variable of range block AMOUNT, WITHDRAWN, CHANGE or LABEL."""
        return self.bits_base + sum(RANGE_WIDTHS[:block])

    def packed_row(self, block):
        """Row (sum 2^k bit_k - value) * ONE = 0 of a range block."""
        return self.row_range + sum(w + 1 for w in RANGE_WIDTHS[:block]) + RANGE_WIDTHS[block]


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
    for block, value in enumerate(({V_AMOUNT: 1}, {V_WITHDRAWN: 1}, change, {V_LABEL: 1})):
        _range_constraints(cs, value, L.bits(block), RANGE_WIDTHS[block])
    cpre = _multi_hash_constraints(cs, [{V_CNULL: 1}, {V_CSECRET: 1}], key, [L.cpre_base, L.cpre_base + P], n_rounds)
    cs.add(cpre, {V_ONE: 1}, {L.cpre_out: 1})
    xs = [{L.cpre_out: 1}, {V_TOKEN: 1}, change, {V_LABEL: 1}]
    ccm = _multi_hash_constraints(cs, xs, key, [L.ccm_base + k * P for k in range(4)], n_rounds)
    cs.add(ccm, {V_ONE: 1}, {V_CHANGE_CM: 1})
    cs.add(lc_add({V_LABEL: 1}, {V_ONE: 1}, {V_ALEAF: R - 1}), {V_ONE: 1}, {})
    _merkle_constraints(cs, L, ASSOC, V_ALEAF, V_AROOT)
    assert cs.n_constraints == L.n_constraints
    return cs


def witness(nullifier, secret, recipient, token, withdrawn, amount, label, siblings, bits, change_nullifier, change_secret,
            assoc_siblings, assoc_bits, n_rounds: int = N_ROUNDS):
    """Full assignment (list of n_vars ints).  bits / assoc_bits: one bit per level, leaf first.  root, association_root,
    nullifier_hash, change_commitment and assoc_leaf are derived.  Every range block holds the low bits of the canonical value
    (mod r) it checks, so an overdraw, a withdrawn value of 2^64 or more, a label or amount out of range, or a label that is
    not a leaf of the provider's tree give an assignment that does not satisfy the R1CS."""
    depth = len(siblings)
    assert len(bits) == len(assoc_siblings) == len(assoc_bits) == depth
    L = Layout(depth, n_rounds)
    P = L.perm
    w = [0] * L.n_vars
    w[V_ONE] = 1
    w[V_RECIP] = recipient % R
    w[V_RSQ] = w[V_RECIP] * w[V_RECIP] % R
    w[V_TOKEN], w[V_WITHDRAWN] = token % R, withdrawn % R
    w[V_NULL], w[V_SECRET], w[V_AMOUNT], w[V_LABEL] = nullifier % R, secret % R, amount % R, label % R
    w[V_CNULL], w[V_CSECRET] = change_nullifier % R, change_secret % R
    w[V_ALEAF] = (w[V_LABEL] + 1) % R
    w[V_NHASH] = _multi_hash_witness(w, [w[V_NULL]], 1, [V_NH_PERM], None, n_rounds)
    pre = _multi_hash_witness(w, [w[V_NULL], w[V_SECRET]], KEY, [L.pre_base, L.pre_base + P], L.pre_out, n_rounds)
    cur = _multi_hash_witness(w, [pre, w[V_TOKEN], w[V_AMOUNT], w[V_LABEL]], KEY, [L.leaf_base + k * P for k in range(4)],
                              L.leaf_out, n_rounds)
    change = (w[V_AMOUNT] - w[V_WITHDRAWN]) % R
    for block, value in enumerate((w[V_AMOUNT], w[V_WITHDRAWN], change, w[V_LABEL])):
        for k in range(RANGE_WIDTHS[block]):
            w[L.bits(block) + k] = (value >> k) & 1
    cpre = _multi_hash_witness(w, [w[V_CNULL], w[V_CSECRET]], KEY, [L.cpre_base, L.cpre_base + P], L.cpre_out, n_rounds)
    w[V_CHANGE_CM] = _multi_hash_witness(w, [cpre, w[V_TOKEN], change, w[V_LABEL]], KEY, [L.ccm_base + k * P for k in range(4)],
                                         None, n_rounds)
    for tree, root, sibs, bs, cur in ((POOL, V_ROOT, siblings, bits, cur), (ASSOC, V_AROOT, assoc_siblings, assoc_bits, w[V_ALEAF])):
        w[root] = levels_witness(w, L, tree, cur, sibs, bs)
    return w


def levels_witness(w, L, tree, cur, sibs, bs):
    """Fill tree `tree`'s level blocks from the leaf value `cur` along (sibs, bs) -> the root it reaches."""
    for l in range(L.depth):
        v = L.level(tree, l)
        sib, bit = sibs[l] % R, bs[l] & 1
        left, right = (sib, cur) if bit else (cur, sib)
        w[v["sib"]], w[v["bit"]], w[v["left"]] = sib, bit, left
        cur = _hash2_witness(w, left, right, v["perm1"], v["perm2"], v["out"], L.n_rounds)
    return cur


class ApprovedTree:
    """The provider's tree of approved labels: leaf label + 1 per approved label, in the order given, in a MerkleTree of the
    pool's depth (every other leaf 0)."""

    def __init__(self, depth: int, labels, n_rounds: int = N_ROUNDS):
        self.tree = MerkleTree(depth, n_rounds)
        self.labels = []
        self.approve(labels)

    def approve(self, labels):
        for label in labels:
            assert 0 <= label < 1 << self.tree.depth and label not in self.labels
            self.labels.append(label)
            self.tree.insert(label + 1)

    def root(self) -> int:
        return self.tree.root()

    def path(self, label):
        """(siblings, bits) of an approved label's leaf."""
        return self.tree.path(self.labels.index(label))
