"""The frozen privacy-pool *association-set withdraw* statement as an R1CS, plus its witness map.

The fourth statement of the library (DESIGN.md section 3); the product's C++ builder
(owshen_b200/csrc/withdraw_circuit.hpp: AssociationBuilder) must reproduce it entry for entry.  An association set
provider publishes the root of a Merkle tree over a subset of the pool's deposits (Buterin, Illum, Nadler, Schaer and
Soleimani, "Blockchain Privacy and Regulatory Compliance: Towards a Practical Equilibrium", 2023); a withdrawer proves that
their note is a leaf of the pool's tree and of that subset's tree, and reveals nothing else.

Statement (public: root, nullifier_hash, recipient, association_root):
  I know (nullifier, secret, siblings[depth], bits[depth], assoc_siblings[depth], assoc_bits[depth]) such that
    nullifier_hash   = MultiMiMC7([nullifier], key=1)                 (the withdraw statement's: one nullifier set)
    commitment       = MultiMiMC7([nullifier, secret], key=0)         (the deposit statement's leaf)
    root             = Merkle root reached from commitment along (siblings, bits)
    association_root = Merkle root reached from commitment along (assoc_siblings, assoc_bits)
                       both with node = MultiMiMC7([left, right], key=0)
  and recipient is bound by recipient^2 = recipient_sq.
Both trees have one depth: with two, a key's shape would fix only their sum, and the prover recognises keys by shape.

Variable layout (index -> meaning), P = 4*n_rounds, a level block is the withdraw statement's (sibling, bit, left,
perm1[P], perm2[P], out), 2P + 4 variables:
  0 ONE | 1 root | 2 nullifier_hash | 3 recipient | 4 association_root        (public, n_pub = 4)
  5 nullifier | 6 secret | 7 recipient_sq
  8 .. 8+P                         nullifier-hash permutation
  then commitment block            perm1[P] perm2[P] out
  then depth pool levels, then depth association levels
Constraint order: recipient; nullifier-hash perm rounds, its output; commitment perm1, perm2, output; per pool level:
boolean, select, perm1, perm2, output; (cur - root) * ONE = 0; the association levels alike, then
(cur - association_root) * ONE = 0.
Sizes: n_vars = 9 + 3P + depth*(4P + 8), n_constraints = 5 + 3P + depth*(4P + 6); with 91 rounds at depth 32 that is
47 949 variables and 47 881 constraints, domain 2^16.
"""
from .bn254 import R
from .mimc7 import N_ROUNDS
from .withdraw_circuit import R1CS, _hash2_constraints, _hash2_witness, _perm_constraints, _perm_witness, lc_add

N_PUB = 4
V_ONE, V_ROOT, V_NHASH, V_RECIP, V_AROOT, V_NULL, V_SECRET, V_RSQ = range(8)
V_NH_PERM = 8
POOL, ASSOC = 0, 1


class Layout:
    def __init__(self, depth: int, n_rounds: int = N_ROUNDS):
        self.depth, self.n_rounds = depth, n_rounds
        P = self.perm = 4 * n_rounds
        self.cm_base = V_NH_PERM + P
        self.cm_out = self.cm_base + 2 * P
        self.lvl_size = 2 * P + 4
        self.tree_base = (self.cm_out + 1, self.cm_out + 1 + depth * self.lvl_size)
        self.n_vars = self.tree_base[ASSOC] + depth * self.lvl_size
        self.n_constraints = 5 + 3 * P + depth * (4 * P + 6)
        assert self.n_vars == 9 + 3 * P + depth * (4 * P + 8)

    def level(self, tree, l):
        b = self.tree_base[tree] + l * self.lvl_size
        P = self.perm
        return dict(sib=b, bit=b + 1, left=b + 2, perm1=b + 3, perm2=b + 3 + P, out=b + 3 + 2 * P)


def build_r1cs(depth: int, n_rounds: int = N_ROUNDS) -> R1CS:
    assert 1 <= depth <= 32
    L = Layout(depth, n_rounds)
    cs = R1CS(L.n_vars, N_PUB)
    cs.add({V_RECIP: 1}, {V_RECIP: 1}, {V_RSQ: 1})
    h = _perm_constraints(cs, {V_NULL: 1}, {V_ONE: 1}, V_NH_PERM, n_rounds)
    cs.add(lc_add({V_ONE: 1}, {V_NULL: 1}, h), {V_ONE: 1}, {V_NHASH: 1})
    _hash2_constraints(cs, {V_NULL: 1}, {V_SECRET: 1}, L.cm_base, L.cm_base + L.perm, L.cm_out, n_rounds)
    for tree, root in ((POOL, V_ROOT), (ASSOC, V_AROOT)):
        cur = L.cm_out
        for l in range(depth):
            v = L.level(tree, l)
            cs.add({v["bit"]: 1}, lc_add({v["bit"]: 1}, {V_ONE: R - 1}), {})
            cs.add({v["bit"]: 1}, lc_add({v["sib"]: 1}, {cur: R - 1}), lc_add({v["left"]: 1}, {cur: R - 1}))
            right = lc_add({v["sib"]: 1}, {cur: 1}, {v["left"]: R - 1})
            _hash2_constraints(cs, {v["left"]: 1}, right, v["perm1"], v["perm2"], v["out"], n_rounds)
            cur = v["out"]
        cs.add(lc_add({cur: 1}, {root: R - 1}), {V_ONE: 1}, {})
    assert cs.n_constraints == L.n_constraints
    return cs


def witness(nullifier, secret, recipient, siblings, bits, assoc_siblings, assoc_bits, n_rounds: int = N_ROUNDS):
    """Full assignment (list of n_vars ints).  bits / assoc_bits: one bit per level, leaf first.  root, nullifier_hash and
    association_root are derived, so a note that is not a leaf of a tree gives a root no provider published."""
    depth = len(siblings)
    assert len(bits) == len(assoc_siblings) == len(assoc_bits) == depth
    L = Layout(depth, n_rounds)
    w = [0] * L.n_vars
    w[V_ONE] = 1
    w[V_RECIP] = recipient % R
    w[V_NULL] = nullifier % R
    w[V_SECRET] = secret % R
    w[V_RSQ] = w[V_RECIP] * w[V_RECIP] % R
    w[V_NHASH] = (1 + w[V_NULL] + _perm_witness(w, w[V_NULL], 1, V_NH_PERM, n_rounds)) % R
    cm = _hash2_witness(w, w[V_NULL], w[V_SECRET], L.cm_base, L.cm_base + L.perm, L.cm_out, n_rounds)
    for tree, root, sibs, bs in ((POOL, V_ROOT, siblings, bits), (ASSOC, V_AROOT, assoc_siblings, assoc_bits)):
        cur = cm
        for l in range(depth):
            v = L.level(tree, l)
            sib, bit = sibs[l] % R, bs[l] & 1
            left, right = (sib, cur) if bit else (cur, sib)
            w[v["sib"]], w[v["bit"]], w[v["left"]] = sib, bit, left
            cur = _hash2_witness(w, left, right, v["perm1"], v["perm2"], v["out"], n_rounds)
        w[root] = cur
    return w
