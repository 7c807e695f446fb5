"""The frozen privacy-pool *owned labeled transfer* statement (two spend-key notes that carry their deposit's label in, two
out, a public withdrawal) as an R1CS, plus its witness map and the owned labeled note format.

The ninth statement of the library (DESIGN.md section 3); the product's C++ builder
(owshen_b200/csrc/withdraw_circuit.hpp: OwnedLabeledTransferBuilder) must reproduce it entry for entry.  It joins the owned
transfer (oracle/owned_circuit.py: only the recipient's spending key can spend an output) and the labeled association
withdrawal (oracle/labeled_association_circuit.py: the deposit's label follows the value, and a provider's approved list
is checked on it), so value can move privately between people and keep its compliance story.

Keys and notes (MultiMiMC7 keys 0..5 are taken; this family adds 6 and 7 and reuses 3 and 5):
  spending key      s; spend public key P = MultiMiMC7([s], 3), the owned transfer's, so one wallet key owns both families
  precommitment     MultiMiMC7([P, blinding], 6); a depositor sends (precommitment, token, amount), which does not reveal P
  leaf              MultiMiMC7([precommitment, token, amount < 2^64, label < 2^32], 7), for a deposit and a transfer output
  nullifier         MultiMiMC7([s, leaf, index], 5), index = the input's pool leaf index from its path bits (the owned
                    nullifier unchanged, so one nullifier set covers every statement)
Keys 6 and 7 keep the leaf apart from the other families: a key-7 leaf does not open as an owned (key 4), labeled (key 2) or
transfer (key 0) note, and their leaves do not open here.  The sender of an output knows P, blinding, the precommitment, the
leaf and its index but not s, which comes first in the nullifier chain and is bound to P by the owner permutation.

The policy:
  one label per transaction: a single private label hashes all four leaves, so both nonzero inputs descend from one deposit
  and the outputs inherit its label by constraint (a zero-value input is not bound to root, so its label does not matter);
  no deposits through the statement: the public amount is withdrawn < 2^64, paid to recipient, and
  in0 + in1 = out0 + out1 + withdrawn with all five values below 2^64 holds over the integers, so two dummy inputs give
  zero outputs; deposits go through the node, which assigns label = pool leaf index (deposit_owned_labeled);
  approval on every spend: assoc_leaf = label + 1 reaches association_root, the ApprovedLabels tree
  (oracle/labeled_association_circuit.py: ApprovedTree) unchanged.

Variable layout (index -> meaning), P = 4*n_rounds, a level block is the withdraw statement's 2P + 4 variables:
  0 ONE | 1 root | 2 association_root | 3 token | 4 withdrawn | 5 recipient | 6, 7 nf[2] | 8, 9 out_cm[2]  (public, n_pub = 9)
  10 recipient_sq | 11 nf_diff_inv | 12 label | 13 assoc_leaf | 14.. label bits (32) | 46.. withdrawn bits (64)
  110.. input blocks 0, 1; each 69 + 10P + depth*(2P + 4) variables:
        +0 spend_key | +1 blinding | +2 amount | +3..+66 amount bits, LSB first
        +67 owner permutation (P; the owner P = 3 + s + hash(s, 3) is a linear combination, not a variable)
        +67+P precommitment perm1, perm2 | +67+3P its output | +68+3P leaf perm[4] | +68+7P its output
        +69+7P depth pool levels | then the nullifier's three permutations (3P; its output row binds nf[i])
  then  output blocks 0, 1; each 69 + 6P variables:
        +0 owner | +1 blinding | +2 amount | +3..+66 amount bits | +67 precommitment perm1, perm2 | +67+2P its output
        +68+2P leaf perm[4] | +68+6P its output
  then  depth association levels
Constraint order:
  recipient^2; the 32-bit range of label, the 64-bit range of withdrawn;
  per input: owner permutation; precommitment perm1, perm2 and its output row; the leaf over (precommitment, token, amount,
             label), its output row; the pool levels; (root - node) * amount = 0; the amount's range; the nullifier's three
             permutations, r3 * ONE = nf[i];
  per output: the amount's range; precommitment; leaf; (leaf_out - out_cm[j]) * ONE = 0;
  (in0 + in1 - out0 - out1 - withdrawn) * ONE = 0; (nf[0] - nf[1]) * nf_diff_inv = ONE; (label + ONE - assoc_leaf) * ONE = 0;
  the association levels, then (cur - association_root) * ONE = 0.
Sizes: n_vars = 386 + 32P + depth*(6P + 12), n_constraints = 377 + 32P + depth*(6P + 9); with 91 rounds at depth 32 that is
82 306 variables and 82 201 constraints, domain 2^17.  No other statement has n_pub 9, so a key's shape names its statement.

Note delivery (oracle/notes.py's scheme): the record of an owned labeled note is the record of the four words (P, blinding,
token, amount + 2^64 label); word 3 is below 2^96 < r, so the record and the envelope keep their size.  A wallet with view key
v and spend public key P owns a record only if it decrypts under v, word 3 is below 2^96, the first word is P and the key-7
leaf of (key-6 precommitment(m0, m1), m2, word 3 mod 2^64, word 3 >> 64) is the commitment.
"""
from . import notes
from .bn254 import R
from .labeled_circuit import _multi_hash_constraints, _multi_hash_witness, _range_constraints, _merkle_constraints
from .mimc7 import N_ROUNDS, multi_hash
from .owned_circuit import OWNER_KEY, NULLIFIER_KEY, nullifier, spend_public_key  # noqa: F401
from .withdraw_circuit import R1CS, _hash2_witness, lc_add

N_PUB = 9
AMOUNT_BITS, LABEL_BITS = 64, 32
PRE_KEY, LEAF_KEY = 6, 7
(V_ONE, V_ROOT, V_AROOT, V_TOKEN, V_WITHDRAWN, V_RECIP) = range(6)
V_NF = (6, 7)
V_OUT_CM = (8, 9)
V_RSQ, V_NF_INV, V_LABEL, V_ALEAF = 10, 11, 12, 13
V_LABEL_BITS = 14
V_WITHDRAWN_BITS = V_LABEL_BITS + LABEL_BITS
V_IN_BASE = V_WITHDRAWN_BITS + AMOUNT_BITS
ASSOC = 2                                   # Layout.level's tree index of the association path (0, 1: the inputs' pool paths)


def precommitment(owner, blinding, n_rounds: int = N_ROUNDS) -> int:
    return multi_hash([owner % R, blinding % R], PRE_KEY, n_rounds)


def leaf(pre, token, amount, label, n_rounds: int = N_ROUNDS) -> int:
    return multi_hash([pre % R, token % R, amount % R, label % R], LEAF_KEY, n_rounds)


def note_leaf(owner, blinding, token, amount, label, n_rounds: int = N_ROUNDS) -> int:
    return leaf(precommitment(owner, blinding, n_rounds), token, amount, label, n_rounds)


class Layout:
    def __init__(self, depth: int, n_rounds: int = N_ROUNDS):
        self.depth, self.n_rounds = depth, n_rounds
        P = self.perm = 4 * n_rounds
        self.lvl_size = 2 * P + 4
        self.in_size = 69 + 10 * P + depth * self.lvl_size
        self.out_size = 69 + 6 * P
        self.out_base = V_IN_BASE + 2 * self.in_size
        self.assoc_base = self.out_base + 2 * self.out_size
        self.n_vars = self.assoc_base + depth * self.lvl_size
        self.n_constraints = 377 + 32 * P + depth * (6 * P + 9)
        assert self.n_vars == 386 + 32 * P + depth * (6 * P + 12)
        if n_rounds == N_ROUNDS:
            assert (self.n_vars, self.n_constraints) == (12034 + 2196 * depth, 12025 + 2193 * depth)
        # named rows, for the soundness tests
        self.row_label_range = LABEL_BITS + 1
        self.row_withdrawn_range = self.row_label_range + AMOUNT_BITS + 1
        in_rows = 10 * P + 69 + depth * (2 * P + 3)
        in0 = self.row_withdrawn_range + 1
        self.row_root = [in0 + i * in_rows + 7 * P + 2 + depth * (2 * P + 3) for i in range(2)]
        self.row_in_range = [r + 65 for r in self.row_root]
        self.row_nf = [in0 + (i + 1) * in_rows - 1 for i in range(2)]
        out_rows = 6 * P + 68
        out0 = in0 + 2 * in_rows
        self.row_out_range = [out0 + j * out_rows + 64 for j in range(2)]
        self.row_out_cm = [out0 + (j + 1) * out_rows - 1 for j in range(2)]
        self.row_balance = out0 + 2 * out_rows
        self.row_nf_diff = self.row_balance + 1
        self.row_assoc_leaf = self.row_balance + 2
        self.row_assoc_root = self.n_constraints - 1

    def note(self, base):
        """Variables of the note block at `base` (input or output): the parts both kinds share."""
        P = self.perm
        return dict(key=base, blinding=base + 1, amount=base + 2, bits=base + 3, pre=base + 67, pre_out=base + 67 + 2 * P,
                    leaf=base + 68 + 2 * P, leaf_out=base + 68 + 6 * P)

    def inp(self, i):
        b = V_IN_BASE + i * self.in_size
        P = self.perm
        v = self.note(b + P)
        v.update(key=b, blinding=b + 1, amount=b + 2, bits=b + 3, owner_perm=b + 67, lvl_base=b + 69 + 7 * P,
                 nf_perm=b + 69 + 7 * P + self.depth * self.lvl_size)
        return v

    def out(self, j):
        return self.note(self.out_base + j * self.out_size)

    def level(self, tree, l):
        """Level l of input 0's or 1's pool path (tree 0, 1) or of the association path (tree ASSOC)."""
        b = (self.inp(tree)["lvl_base"] if tree < 2 else self.assoc_base) + l * self.lvl_size
        P = self.perm
        return dict(sib=b, bit=b + 1, left=b + 2, perm1=b + 3, perm2=b + 3 + P, out=b + 3 + 2 * P)


def _note_constraints(cs, owner_lc, v, P, n_rounds):
    pre = _multi_hash_constraints(cs, [owner_lc, {v["blinding"]: 1}], {V_ONE: PRE_KEY}, [v["pre"], v["pre"] + P], n_rounds)
    cs.add(pre, {V_ONE: 1}, {v["pre_out"]: 1})
    xs = [{v["pre_out"]: 1}, {V_TOKEN: 1}, {v["amount"]: 1}, {V_LABEL: 1}]
    lf = _multi_hash_constraints(cs, xs, {V_ONE: LEAF_KEY}, [v["leaf"] + k * P for k in range(4)], n_rounds)
    cs.add(lf, {V_ONE: 1}, {v["leaf_out"]: 1})


def build_r1cs(depth: int, n_rounds: int = N_ROUNDS) -> R1CS:
    assert 1 <= depth <= 32
    L = Layout(depth, n_rounds)
    P = L.perm
    cs = R1CS(L.n_vars, N_PUB)
    cs.add({V_RECIP: 1}, {V_RECIP: 1}, {V_RSQ: 1})
    _range_constraints(cs, {V_LABEL: 1}, V_LABEL_BITS, LABEL_BITS)
    _range_constraints(cs, {V_WITHDRAWN: 1}, V_WITHDRAWN_BITS, AMOUNT_BITS)
    for i in range(2):
        v = L.inp(i)
        s = {v["key"]: 1}
        owner = _multi_hash_constraints(cs, [s], {V_ONE: OWNER_KEY}, [v["owner_perm"]], n_rounds)
        _note_constraints(cs, owner, v, P, n_rounds)
        cur = v["leaf_out"]
        index = {}
        for l in range(depth):
            lv = L.level(i, l)
            cs.add({lv["bit"]: 1}, lc_add({lv["bit"]: 1}, {V_ONE: R - 1}), {})
            cs.add({lv["bit"]: 1}, lc_add({lv["sib"]: 1}, {cur: R - 1}), lc_add({lv["left"]: 1}, {cur: R - 1}))
            right = lc_add({lv["sib"]: 1}, {cur: 1}, {lv["left"]: R - 1})
            r2 = _multi_hash_constraints(cs, [{lv["left"]: 1}, right], {}, [lv["perm1"], lv["perm2"]], n_rounds)
            cs.add(r2, {V_ONE: 1}, {lv["out"]: 1})
            cur = lv["out"]
            index[lv["bit"]] = pow(2, l, R)
        cs.add(lc_add({V_ROOT: 1}, {cur: R - 1}), {v["amount"]: 1}, {})
        _range_constraints(cs, {v["amount"]: 1}, v["bits"], AMOUNT_BITS)
        nf = _multi_hash_constraints(cs, [s, {v["leaf_out"]: 1}, index], {V_ONE: NULLIFIER_KEY},
                                     [v["nf_perm"] + k * P for k in range(3)], n_rounds)
        cs.add(nf, {V_ONE: 1}, {V_NF[i]: 1})
    for j in range(2):
        v = L.out(j)
        _range_constraints(cs, {v["amount"]: 1}, v["bits"], AMOUNT_BITS)
        _note_constraints(cs, {v["key"]: 1}, v, P, n_rounds)
        cs.add(lc_add({v["leaf_out"]: 1}, {V_OUT_CM[j]: R - 1}), {V_ONE: 1}, {})
    i0, i1, o0, o1 = L.inp(0)["amount"], L.inp(1)["amount"], L.out(0)["amount"], L.out(1)["amount"]
    cs.add({i0: 1, i1: 1, o0: R - 1, o1: R - 1, V_WITHDRAWN: R - 1}, {V_ONE: 1}, {})
    cs.add({V_NF[0]: 1, V_NF[1]: R - 1}, {V_NF_INV: 1}, {V_ONE: 1})
    cs.add(lc_add({V_LABEL: 1}, {V_ONE: 1}, {V_ALEAF: R - 1}), {V_ONE: 1}, {})
    _merkle_constraints(cs, L, ASSOC, V_ALEAF, V_AROOT)
    assert cs.n_constraints == L.n_constraints
    return cs


def _levels_witness(w, L, tree, cur, sibs, bits):
    for l in range(L.depth):
        v = L.level(tree, l)
        sib, bit = sibs[l] % R, (bits >> l) & 1
        left, right = (sib, cur) if bit else (cur, sib)
        w[v["sib"]], w[v["bit"]], w[v["left"]] = sib, bit, left
        cur = _hash2_witness(w, left, right, v["perm1"], v["perm2"], v["out"], L.n_rounds)
    return cur


def _note_witness(w, v, first, owner, blinding, amount, P, n_rounds):
    """Fills a note block's first variable (the spend key of an input, the owner of an output), blinding, amount, its low 64
    bits, the precommitment and the leaf under w's token and label; returns the leaf."""
    w[v["key"]], w[v["blinding"]], w[v["amount"]] = first % R, blinding % R, amount
    for k in range(AMOUNT_BITS):
        w[v["bits"] + k] = (amount >> k) & 1
    pre = _multi_hash_witness(w, [owner % R, w[v["blinding"]]], PRE_KEY, [v["pre"], v["pre"] + P], v["pre_out"], n_rounds)
    return _multi_hash_witness(w, [pre, w[V_TOKEN], amount, w[V_LABEL]], LEAF_KEY, [v["leaf"] + k * P for k in range(4)],
                               v["leaf_out"], n_rounds)


def witness(root, token, withdrawn, recipient, label, inputs, outputs, assoc_siblings, assoc_bits, n_rounds: int = N_ROUNDS):
    """Full assignment (list of n_vars ints).
    inputs: two (spend_key, blinding, amount, siblings[depth], path_bits); outputs: two (owner, blinding, amount);
    path_bits and assoc_bits are words, bit l for level l.  root is the caller's; association_root, the nullifiers, the output
    leaves and assoc_leaf are derived.  The label and withdrawn bits are the low bits of their canonical values, so a wrong
    spend key, an input of nonzero value off the tree or under another label, an unapproved label, an overdraw, two inputs
    with one nullifier, or a label or withdrawn value out of range give an assignment that does not satisfy the R1CS."""
    depth = len(assoc_siblings)
    assert all(len(n[3]) == depth for n in inputs)
    assert all(0 <= n[2] < 1 << AMOUNT_BITS for n in list(inputs) + list(outputs)), "amounts are below 2^64"
    L = Layout(depth, n_rounds)
    P = L.perm
    w = [0] * L.n_vars
    w[V_ONE] = 1
    w[V_ROOT], w[V_TOKEN], w[V_WITHDRAWN] = root % R, token % R, withdrawn % R
    w[V_RECIP] = recipient % R
    w[V_RSQ] = w[V_RECIP] * w[V_RECIP] % R
    w[V_LABEL] = label % R
    w[V_ALEAF] = (w[V_LABEL] + 1) % R
    for k in range(LABEL_BITS):
        w[V_LABEL_BITS + k] = (w[V_LABEL] >> k) & 1
    for k in range(AMOUNT_BITS):
        w[V_WITHDRAWN_BITS + k] = (w[V_WITHDRAWN] >> k) & 1
    for i, (s, blinding, amount, sibs, bits) in enumerate(inputs):
        v = L.inp(i)
        s %= R
        owner = _multi_hash_witness(w, [s], OWNER_KEY, [v["owner_perm"]], None, n_rounds)
        lf = _note_witness(w, v, s, owner, blinding, amount, P, n_rounds)
        _levels_witness(w, L, i, lf, sibs, bits)
        index = bits & ((1 << depth) - 1)
        w[V_NF[i]] = _multi_hash_witness(w, [s, lf, index], NULLIFIER_KEY, [v["nf_perm"] + k * P for k in range(3)], None,
                                         n_rounds)
    for j, (owner, blinding, amount) in enumerate(outputs):
        w[V_OUT_CM[j]] = _note_witness(w, L.out(j), owner, owner, blinding, amount, P, n_rounds)
    d = (w[V_NF[0]] - w[V_NF[1]]) % R
    w[V_NF_INV] = pow(d, R - 2, R) if d else 0
    w[V_AROOT] = _levels_witness(w, L, ASSOC, w[V_ALEAF], assoc_siblings, assoc_bits)
    return w


# ---- note delivery --------------------------------------------------------------------------------------------------------
def pack_words(note):
    """The four record words of an owned labeled note (owner, blinding, token, amount, label)."""
    owner, blinding, token, amount, label = note
    assert 0 <= amount < 1 << AMOUNT_BITS and 0 <= label < 1 << LABEL_BITS
    return (owner, blinding, token, amount + (label << AMOUNT_BITS))


def unpack_words(m):
    """(owner, blinding, token, amount, label) from four decrypted words, or None when word 3 is 2^96 or more."""
    if m[3] >> (AMOUNT_BITS + LABEL_BITS):
        return None
    return (m[0], m[1], m[2], m[3] & ((1 << AMOUNT_BITS) - 1), m[3] >> AMOUNT_BITS)


def encrypt_note(pk, note, e):
    """-> (status, record, commitment) of an owned labeled note (owner, blinding, token, amount, label) to the view address
    pk: notes.encrypt's scheme over pack_words(note), and the note's key-7 leaf as the commitment."""
    m = pack_words(note)
    assert all(0 <= x < R for x in m[:3] + (pk[0], e))
    fail = lambda st: (st, bytes(notes.RECORD_BYTES), 0)
    V = notes.decompress_or_none(*pk)
    if V is None:
        return fail(notes.ENC_BAD_KEY)
    Vp = notes.clear_cofactor(V)
    if Vp == notes.IDENTITY:
        return fail(notes.ENC_BAD_KEY)
    if e % notes.L == 0:
        return fail(notes.ENC_BAD_EPHEMERAL)
    E = notes.mul(notes.bjj.BASE, e)
    k = notes._key(notes.mul(Vp, e))
    cs = [(x + notes._pad(i, k)) % R for i, x in enumerate(m)]
    return notes.ENC_OK, notes.encode_record(E[0], E[1] & 1, cs), note_leaf(*note)


def scan_notes(view_keys, spend_public_keys, records, commitments):
    """-> (owners, plaintexts) as notes.scan, key j being (view_keys[j], spend_public_keys[j]) and owning a record only if
    word 3 is below 2^96, the first word is spend_public_keys[j] and the note's key-7 leaf matches.  A plaintext is the four
    decrypted words (word 3 = amount + 2^64 label)."""
    owners, plain = [], []
    for rec, cm in zip(records, commitments):
        p = notes.prepare(rec, cm)
        owner, m_owned = (notes.MALFORMED, None) if p is None else (notes.NOT_OWNED, None)
        if p is not None:
            Ep, cs = p
            for j, (v, P) in enumerate(zip(view_keys, spend_public_keys)):
                k = notes._key(notes.mul(Ep, v))
                m = [(c - notes._pad(i, k)) % R for i, c in enumerate(cs)]
                note = unpack_words(m)
                if note is not None and m[0] == P and note_leaf(*note) == cm:
                    owner, m_owned = j, m
                    break
        owners.append(owner)
        plain.append(bytes(notes.PLAINTEXT_BYTES) if m_owned is None else b"".join(x.to_bytes(32, "little") for x in m_owned))
    return owners, plain
