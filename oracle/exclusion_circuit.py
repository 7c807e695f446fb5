"""The frozen privacy-pool *exclusion withdraw* statement as an R1CS, plus its witness map and the blocklist tree.

The fifth statement of the library (DESIGN.md section 3); the product's C++ builder
(owshen_b200/csrc/withdraw_circuit.hpp: ExclusionBuilder) must reproduce it entry for entry.  A compliance provider publishes
the root of a tree over a blocklist of flagged deposits; a withdrawer proves that their note is a leaf of the pool's tree and
that its deposit is not on the list, and reveals nothing else (the exclusion half of Buterin, Illum, Nadler, Schaer and
Soleimani, "Blockchain Privacy and Regulatory Compliance: Towards a Practical Equilibrium", 2023).

The blocklist names deposits by their leaf index in the pool tree (public: the order of the deposits).  The index is
already in the witness as sum 2^l bit_l over the pool path's boolean bits, so excluding it needs 33-bit range checks only;
keying by commitment would need full 254-bit comparisons.  Flagged indices i_1 < ... < i_n in [0, 2^depth) give the keys
k_0 = 0, k_j = i_j + 1, k_{n+1} = 2^32 + 1, and leaf j = MultiMiMC7([k_j, k_{j+1}], 0) for j = 0..n, placed in order in a
tree of the pool's depth (other leaves 0, as mimc7.MerkleTree).  A note at index i, x = i + 1, is unflagged exactly when
some leaf brackets it: k_j < x < k_{j+1}.

Statement (public: root, nullifier_hash, recipient, exclusion_root):
  I know (nullifier, secret, siblings[depth], bits[depth], low, next, excl_siblings[depth], excl_bits[depth]) such that
    the withdraw statement holds for (root, nullifier_hash, recipient) (one nullifier set for all withdraw statements);
    x = ONE + sum_l 2^l bits[l];
    low, next, gap_lo = x - low - 1 and gap_hi = next - x - 1 are each below 2^33;
    exclusion_root = Merkle root reached from MultiMiMC7([low, next], 0) along (excl_siblings, excl_bits).
Sound because low, next < 2^33 and x <= 2^32: x - low - 1 is below 2^33 exactly when x > low, otherwise it is about
r - 2^33 (mod r); likewise for next.  An empty leaf (0) has no known preimage; the path length is fixed, so no internal node
stands in for a leaf.

Variable layout (index -> meaning), P = 4*n_rounds, a level block is the withdraw statement's 2P + 4 variables:
  0 ONE | 1 root | 2 nullifier_hash | 3 recipient | 4 exclusion_root        (public, n_pub = 4)
  5 nullifier | 6 secret | 7 recipient_sq | 8 low | 9 next
  10 .. 10+P                       nullifier-hash permutation
  then commitment block            perm1[P] perm2[P] out
  then depth pool levels
  then low bits[33] | next bits[33] | gap_lo bits[33] | gap_hi bits[33]     (LSB first)
  then leaf block                  perm1[P] perm2[P] out
  then depth exclusion levels
Constraint order: recipient; nullifier-hash perm rounds, its output; commitment perm1, perm2, output; per pool level:
boolean, select, perm1, perm2, output; (cur - root) * ONE = 0; the four range checks (33 rows bit * (bit - ONE) = 0, then
(sum 2^k bit_k - value) * ONE = 0) of low, next, gap_lo, gap_hi; the leaf's perm1, perm2, output; the exclusion levels, then
(cur - exclusion_root) * ONE = 0.
Sizes: n_vars = 144 + 5P + depth*(4P + 8), n_constraints = 142 + 5P + depth*(4P + 6); with 91 rounds at depth 32 that is
48 812 variables and 48 746 constraints, domain 2^16.
"""
import bisect

from .bn254 import R
from .mimc7 import N_ROUNDS, MerkleTree, hash2
from .withdraw_circuit import R1CS, _hash2_constraints, _hash2_witness, _perm_constraints, _perm_witness, lc_add, lc_scale

N_PUB = 4
RANGE_BITS = 33
KEY_MAX = (1 << 32) + 1                     # k_{n+1}: above every x = index + 1 <= 2^32
V_ONE, V_ROOT, V_NHASH, V_RECIP, V_XROOT, V_NULL, V_SECRET, V_RSQ, V_LOW, V_NEXT = range(10)
V_NH_PERM = 10
POOL, EXCL = 0, 1
LOW, NEXT, GAP_LO, GAP_HI = range(4)


class Layout:
    def __init__(self, depth: int, n_rounds: int = N_ROUNDS):
        self.depth, self.n_rounds = depth, n_rounds
        P = self.perm = 4 * n_rounds
        self.cm_base = V_NH_PERM + P
        self.cm_out = self.cm_base + 2 * P
        self.lvl_size = 2 * P + 4
        self.pool_base = self.cm_out + 1
        self.bits_base = self.pool_base + depth * self.lvl_size
        self.leaf_base = self.bits_base + 4 * RANGE_BITS
        self.leaf_out = self.leaf_base + 2 * P
        self.excl_base = self.leaf_out + 1
        self.tree_base = (self.pool_base, self.excl_base)
        self.n_vars = self.excl_base + depth * self.lvl_size
        self.n_constraints = 142 + 5 * P + depth * (4 * P + 6)
        assert self.n_vars == 144 + 5 * P + depth * (4 * P + 8)
        if n_rounds == N_ROUNDS:
            assert (self.n_vars, self.n_constraints) == (1964 + 1464 * depth, 1962 + 1462 * depth)

    def level(self, tree, l):
        b = self.tree_base[tree] + l * self.lvl_size
        P = self.perm
        return dict(sib=b, bit=b + 1, left=b + 2, perm1=b + 3, perm2=b + 3 + P, out=b + 3 + 2 * P)

    def bits(self, block):
        """First variable of range block LOW, NEXT, GAP_LO or GAP_HI."""
        return self.bits_base + block * RANGE_BITS


def _range_constraints(cs, value, bits, n_bits):
    """n_bits rows bit_k * (bit_k - ONE) = 0, then (sum 2^k bit_k - value) * ONE = 0; value is an LC."""
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
    cs = R1CS(L.n_vars, N_PUB)
    cs.add({V_RECIP: 1}, {V_RECIP: 1}, {V_RSQ: 1})
    h = _perm_constraints(cs, {V_NULL: 1}, {V_ONE: 1}, V_NH_PERM, n_rounds)
    cs.add(lc_add({V_ONE: 1}, {V_NULL: 1}, h), {V_ONE: 1}, {V_NHASH: 1})
    _hash2_constraints(cs, {V_NULL: 1}, {V_SECRET: 1}, L.cm_base, L.cm_base + L.perm, L.cm_out, n_rounds)
    _merkle_constraints(cs, L, POOL, L.cm_out, V_ROOT)
    x = lc_add({V_ONE: 1}, {L.level(POOL, l)["bit"]: pow(2, l, R) for l in range(depth)})
    _range_constraints(cs, {V_LOW: 1}, L.bits(LOW), RANGE_BITS)
    _range_constraints(cs, {V_NEXT: 1}, L.bits(NEXT), RANGE_BITS)
    _range_constraints(cs, lc_add(x, {V_LOW: R - 1}, {V_ONE: R - 1}), L.bits(GAP_LO), RANGE_BITS)
    _range_constraints(cs, lc_add({V_NEXT: 1}, lc_scale(x, R - 1), {V_ONE: R - 1}), L.bits(GAP_HI), RANGE_BITS)
    _hash2_constraints(cs, {V_LOW: 1}, {V_NEXT: 1}, L.leaf_base, L.leaf_base + L.perm, L.leaf_out, n_rounds)
    _merkle_constraints(cs, L, EXCL, L.leaf_out, V_XROOT)
    assert cs.n_constraints == L.n_constraints
    return cs


def witness(nullifier, secret, recipient, siblings, bits, low, next_, excl_siblings, excl_bits, n_rounds: int = N_ROUNDS):
    """Full assignment (list of n_vars ints).  bits / excl_bits: one bit per level, leaf first.  root and exclusion_root are
    derived; the low and next bits are the 33 low bits of low and next, the gap bits the 33 low bits of the canonical
    (x - low - 1) mod r and (next - x - 1) mod r.  A flagged note, a leaf that does not bracket the note, or low / next of
    2^33 or more therefore give an assignment that does not satisfy the R1CS."""
    depth = len(siblings)
    assert len(bits) == len(excl_siblings) == len(excl_bits) == depth
    L = Layout(depth, n_rounds)
    w = [0] * L.n_vars
    w[V_ONE] = 1
    w[V_RECIP] = recipient % R
    w[V_NULL] = nullifier % R
    w[V_SECRET] = secret % R
    w[V_RSQ] = w[V_RECIP] * w[V_RECIP] % R
    w[V_LOW], w[V_NEXT] = low % R, next_ % R
    w[V_NHASH] = (1 + w[V_NULL] + _perm_witness(w, w[V_NULL], 1, V_NH_PERM, n_rounds)) % R
    cm = _hash2_witness(w, w[V_NULL], w[V_SECRET], L.cm_base, L.cm_base + L.perm, L.cm_out, n_rounds)
    leaf = None
    for tree, root, sibs, bs in ((POOL, V_ROOT, siblings, bits), (EXCL, V_XROOT, excl_siblings, excl_bits)):
        if tree == EXCL:
            x = 1 + sum((b & 1) << l for l, b in enumerate(bits))
            for block, value in ((LOW, low), (NEXT, next_), (GAP_LO, (x - low - 1) % R), (GAP_HI, (next_ - x - 1) % R)):
                for k in range(RANGE_BITS):
                    w[L.bits(block) + k] = (value >> k) & 1
            leaf = _hash2_witness(w, w[V_LOW], w[V_NEXT], L.leaf_base, L.leaf_base + L.perm, L.leaf_out, n_rounds)
        cur = cm if tree == POOL else leaf
        for l in range(depth):
            v = L.level(tree, l)
            sib, bit = sibs[l] % R, bs[l] & 1
            left, right = (sib, cur) if bit else (cur, sib)
            w[v["sib"]], w[v["bit"]], w[v["left"]] = sib, bit, left
            cur = _hash2_witness(w, left, right, v["perm1"], v["perm2"], v["out"], n_rounds)
        w[root] = cur
    return w


# ---- the blocklist tree ------------------------------------------------------------------------------------------------
def keys(flagged):
    """k_0 = 0, k_j = i_j + 1 over the sorted distinct flagged indices, k_{n+1} = 2^32 + 1."""
    return [0] + [i + 1 for i in sorted(set(flagged))] + [KEY_MAX]


def leaves(flagged):
    """Leaf j = MultiMiMC7([k_j, k_{j+1}], 0) for j = 0..n."""
    k = keys(flagged)
    return [hash2(a, b) for a, b in zip(k, k[1:])]


class BlocklistTree:
    """The provider's tree over a blocklist of pool leaf indices, depth = the pool tree's."""

    def __init__(self, depth: int, flagged):
        self.depth = depth
        self.flagged = sorted(set(flagged))
        assert all(0 <= i < 1 << depth for i in self.flagged), "flagged indices are pool leaf indices"
        assert len(self.flagged) < 1 << depth, "a tree of depth d holds at most 2^d - 1 flagged indices"
        self.keys = keys(self.flagged)
        self.tree = MerkleTree(depth)
        for leaf in leaves(self.flagged):
            self.tree.insert(leaf)

    def root(self) -> int:
        return self.tree.root()

    def bracket(self, index: int) -> int:
        """The leaf j with k_j < index + 1 < k_{j+1}; ValueError when the index is flagged."""
        x = index + 1
        j = bisect.bisect_left(self.keys, x) - 1
        if self.keys[j + 1] == x:
            raise ValueError(f"pool leaf {index} is on the blocklist")
        return j

    def witness(self, index: int):
        """(low, next, excl_siblings, excl_bits) of an unflagged pool leaf index."""
        j = self.bracket(index)
        sibs, bits = self.tree.path(j)
        return self.keys[j], self.keys[j + 1], sibs, bits
