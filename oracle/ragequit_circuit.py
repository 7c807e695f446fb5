"""The frozen privacy-pool *ragequit* statement (one owned labeled note spent whole, in public, without a provider's
approval) as an R1CS, plus its witness map.

The tenth statement of the library (DESIGN.md section 3); the product's C++ builder
(owshen_b200/csrc/withdraw_circuit.hpp: RagequitBuilder) must reproduce it entry for entry.  Every spend of an owned labeled
note through the owned labeled transfer (oracle/owned_labeled_circuit.py) proves its label is on a provider's approved list,
so without another exit the value of a deposit the provider never approves, or later drops, could not move at all.  The
ragequit is that exit, as in the Privacy Pools design: the holder gives up privacy and takes the note out in public, linked
to its deposit, so the value never joins the approved anonymity set.

Keys and notes: the owned labeled family's, unchanged, and no new MultiMiMC7 key:
  spend public key  P = MultiMiMC7([s], 3)
  precommitment     MultiMiMC7([P, blinding], 6)
  leaf              MultiMiMC7([precommitment, token, amount, label], 7)
  nullifier         MultiMiMC7([s, leaf, index], 5), index = sum 2^l bit_l over the low `depth` path bits: the owned labeled
                    transfer's nullifier bit for bit, so with one nullifier set a note that has been ragequit cannot be
                    transferred later, and a note that has been transferred cannot be ragequit.

Statement (public: root, token, amount, label, recipient, nullifier):
  I know (spend_key, blinding, siblings[depth], bits[depth]) such that the leaf of (MultiMiMC7([spend_key], 3), blinding,
  token, amount, label) reaches root along (siblings, bits) and nullifier is its nullifier; recipient is bound by
  recipient^2 = recipient_sq.

The policy, and why it is sound:
  ownership: the owned transfer's argument.  The leaf reaches root, the leaf fixes the precommitment and so P, and the
    prover must know s with MultiMiMC7([s], 3) = P.  The sender of a note knows P, blinding, the leaf and its index but not
    s, and every guess of s fails the root row.  root is the caller's, so a wrong spend key gives a proof that does not
    verify rather than a proof about another root.
  amount, label and token are bound by the leaf, and need no range rows: both ways a key-7 leaf enters the tree range-check
    them.  deposit_owned_labeled takes u64 amounts and assigns label = the pool leaf index, and the owned labeled transfer
    range-checks its outputs' amounts in-circuit under a 32-bit-checked label.  So a leaf that opens under root has an
    amount below 2^64 and a label below 2^32, and a public amount or label outside those ranges opens no leaf.
  any holder of any owned labeled note may ragequit it, approved or not.  The exit publishes the label, so it is linked to
    its deposit exactly as if the value had never entered the pool.  The note is spent whole: no change, no partial amount.
  the root row is (root - node) * ONE = 0, unconditional (the transfers multiply by the amount so that a zero-value dummy
    input need not open), so a zero-value note off the tree cannot ragequit.
  domain separation: key-0 transfer, key-2 labeled and key-4 owned leaves do not open here, because the leaf key is 7.
  Node-side policy is not in the proof: paying only the original depositor's address, allowing ragequit only for
  unapproved labels, or delays are the node's decisions, taken from the public inputs.

Variable layout (index -> meaning), P = 4*n_rounds, a level block is the withdraw statement's 2P + 4 variables:
  0 ONE | 1 root | 2 token | 3 amount | 4 label | 5 recipient | 6 nullifier                       (public, n_pub = 6)
  7 recipient_sq | 8 spend_key | 9 blinding
  10     owner permutation (P; the owner P = 3 + s + hash(s, 3) is a linear combination, not a variable)
  10+P   precommitment perm1, perm2 (2P) | 10+3P its output
  11+3P  leaf perm[4] (4P) | 11+7P its output
  12+7P  depth pool levels
  then   the nullifier's three permutations (3P; its output row binds nullifier)
Constraint order:
  recipient^2; the owner permutation; the precommitment's two permutations and its output row; the leaf over (pre_out,
  token, amount, label), the public variables entering directly, and its output row; per pool level: boolean, select,
  perm1, perm2, output; (root - node) * ONE = 0; the nullifier's three permutations, r3 * ONE = nullifier.
Sizes: n_vars = 12 + 10P + depth*(2P + 4), n_constraints = 5 + 10P + depth*(2P + 3); with 91 rounds at depth 32 that is
27 076 variables and 27 037 constraints, domain 2^15.  No other statement has n_pub 6, so a key's shape names its statement.
"""
from .bn254 import R
from .labeled_circuit import _multi_hash_constraints, _multi_hash_witness
from .mimc7 import N_ROUNDS
from .owned_circuit import NULLIFIER_KEY, OWNER_KEY
from .owned_labeled_circuit import LEAF_KEY, PRE_KEY, note_leaf, spend_public_key  # noqa: F401
from .withdraw_circuit import R1CS, _hash2_witness, lc_add

N_PUB = 6
V_ONE, V_ROOT, V_TOKEN, V_AMOUNT, V_LABEL, V_RECIP, V_NF, V_RSQ, V_KEY, V_BLINDING = range(10)
V_OWNER_PERM = 10


class Layout:
    def __init__(self, depth: int, n_rounds: int = N_ROUNDS):
        self.depth, self.n_rounds = depth, n_rounds
        P = self.perm = 4 * n_rounds
        self.lvl_size = 2 * P + 4
        self.pre = V_OWNER_PERM + P
        self.pre_out = self.pre + 2 * P
        self.leaf = self.pre_out + 1
        self.leaf_out = self.leaf + 4 * P
        self.lvl_base = self.leaf_out + 1
        self.nf_perm = self.lvl_base + depth * self.lvl_size
        self.n_vars = self.nf_perm + 3 * P
        self.n_constraints = 5 + 10 * P + depth * (2 * P + 3)
        assert self.n_vars == 12 + 10 * P + depth * (2 * P + 4)
        if n_rounds == N_ROUNDS:
            assert (self.n_vars, self.n_constraints) == (3652 + 732 * depth, 3645 + 731 * depth)
        # named rows, for the soundness tests
        self.row_root = 7 * P + 3 + depth * (2 * P + 3)
        self.row_nf = self.n_constraints - 1

    def level(self, l):
        b = self.lvl_base + l * self.lvl_size
        P = self.perm
        return dict(sib=b, bit=b + 1, left=b + 2, perm1=b + 3, perm2=b + 3 + P, out=b + 3 + 2 * P)


def build_r1cs(depth: int, n_rounds: int = N_ROUNDS) -> R1CS:
    assert 1 <= depth <= 32
    L = Layout(depth, n_rounds)
    P = L.perm
    cs = R1CS(L.n_vars, N_PUB)
    cs.add({V_RECIP: 1}, {V_RECIP: 1}, {V_RSQ: 1})
    s = {V_KEY: 1}
    owner = _multi_hash_constraints(cs, [s], {V_ONE: OWNER_KEY}, [V_OWNER_PERM], n_rounds)
    pre = _multi_hash_constraints(cs, [owner, {V_BLINDING: 1}], {V_ONE: PRE_KEY}, [L.pre, L.pre + P], n_rounds)
    cs.add(pre, {V_ONE: 1}, {L.pre_out: 1})
    xs = [{L.pre_out: 1}, {V_TOKEN: 1}, {V_AMOUNT: 1}, {V_LABEL: 1}]
    lf = _multi_hash_constraints(cs, xs, {V_ONE: LEAF_KEY}, [L.leaf + k * P for k in range(4)], n_rounds)
    cs.add(lf, {V_ONE: 1}, {L.leaf_out: 1})
    cur = L.leaf_out
    index = {}
    for l in range(depth):
        lv = L.level(l)
        cs.add({lv["bit"]: 1}, lc_add({lv["bit"]: 1}, {V_ONE: R - 1}), {})
        cs.add({lv["bit"]: 1}, lc_add({lv["sib"]: 1}, {cur: R - 1}), lc_add({lv["left"]: 1}, {cur: R - 1}))
        right = lc_add({lv["sib"]: 1}, {cur: 1}, {lv["left"]: R - 1})
        r2 = _multi_hash_constraints(cs, [{lv["left"]: 1}, right], {}, [lv["perm1"], lv["perm2"]], n_rounds)
        cs.add(r2, {V_ONE: 1}, {lv["out"]: 1})
        cur = lv["out"]
        index[lv["bit"]] = pow(2, l, R)
    cs.add(lc_add({V_ROOT: 1}, {cur: R - 1}), {V_ONE: 1}, {})
    nf = _multi_hash_constraints(cs, [s, {L.leaf_out: 1}, index], {V_ONE: NULLIFIER_KEY}, [L.nf_perm + k * P for k in range(3)],
                                 n_rounds)
    cs.add(nf, {V_ONE: 1}, {V_NF: 1})
    assert cs.n_constraints == L.n_constraints
    return cs


def witness(root, token, amount, label, recipient, spend_key, blinding, siblings, path_bits, n_rounds: int = N_ROUNDS):
    """Full assignment (list of n_vars ints).  path_bits is a word, bit l for level l; only its low depth bits count.  root
    is the caller's; the nullifier is derived.  A wrong spend key, blinding, token, amount, label or path gives an
    assignment that fails the root row."""
    depth = len(siblings)
    L = Layout(depth, n_rounds)
    P = L.perm
    w = [0] * L.n_vars
    w[V_ONE] = 1
    w[V_ROOT], w[V_TOKEN], w[V_AMOUNT], w[V_LABEL] = root % R, token % R, amount % R, label % R
    w[V_RECIP] = recipient % R
    w[V_RSQ] = w[V_RECIP] * w[V_RECIP] % R
    s = w[V_KEY] = spend_key % R
    w[V_BLINDING] = blinding % R
    owner = _multi_hash_witness(w, [s], OWNER_KEY, [V_OWNER_PERM], None, n_rounds)
    pre = _multi_hash_witness(w, [owner, w[V_BLINDING]], PRE_KEY, [L.pre, L.pre + P], L.pre_out, n_rounds)
    cur = lf = _multi_hash_witness(w, [pre, w[V_TOKEN], w[V_AMOUNT], w[V_LABEL]], LEAF_KEY, [L.leaf + k * P for k in range(4)],
                                   L.leaf_out, n_rounds)
    for l in range(depth):
        v = L.level(l)
        sib, bit = siblings[l] % R, (path_bits >> l) & 1
        left, right = (sib, cur) if bit else (cur, sib)
        w[v["sib"]], w[v["bit"]], w[v["left"]] = sib, bit, left
        cur = _hash2_witness(w, left, right, v["perm1"], v["perm2"], v["out"], n_rounds)
    index = path_bits & ((1 << depth) - 1)
    w[V_NF] = _multi_hash_witness(w, [s, lf, index], NULLIFIER_KEY, [L.nf_perm + k * P for k in range(3)], None, n_rounds)
    return w
