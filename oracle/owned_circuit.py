"""The frozen privacy-pool *owned transfer* statement (two spend-key notes in, two out, a public amount) as an R1CS, plus its
witness map and the spend-key note format.

The eighth statement of the library (DESIGN.md section 3); the product's C++ builder
(owshen_b200/csrc/withdraw_circuit.hpp: OwnedTransferBuilder) must reproduce it entry for entry.  A transfer note
(oracle/transfer_circuit.py) is spendable by whoever knows its nullifier and secret, and the sender picks both, so a sender
can spend what they send.  An owned note is bound to the recipient's spending key instead: only the holder of s can open
its nullifier.

Keys and notes (MultiMiMC7 keys 0: commitments and Merkle nodes, 1: nullifier hashes, 2: labeled notes are taken):
  spending key      s, a canonical Fr element kept by the wallet
  spend public key  P = MultiMiMC7([s], key=3)
  address           (P, V) with V the view key's BabyJubJub address (oracle/notes.py); the two keys are separate, so a
                    view key sees incoming notes but can neither spend them nor compute their nullifiers
  note              (P, blinding, token, amount < 2^64)
  commitment        cm = MultiMiMC7([P, blinding, token, amount], key=4)
  nullifier         MultiMiMC7([s, cm, index], key=5), index = sum 2^l bit_l over the input's path bits (its leaf index)
Key 4 keeps owned leaves apart from transfer commitments: under key 0 the leaf would be a transfer note with nullifier = P
and secret = blinding, both known to the sender.  s comes first in the nullifier chain, so the chain never passes through P
and knowing (P, cm, index) does not give the nullifier.  The index makes two deposits of one note two spendable notes.

Statement (public: root, public_amount, token, recipient, nullifier[2], out_commitment[2]; the transfer's interface):
  I know two input notes (s, blinding, amount, siblings[depth], bits[depth]) and two output notes (P_out, blinding, amount)
  of `token` such that
    nullifier[i] = MultiMiMC7([s_i, cm_i, index_i], 5) with cm_i the commitment of (MultiMiMC7([s_i], 3), blinding_i, token,
                   amount_i), and the two nullifiers differ;
    every nonzero-valued input's commitment reaches root along its Merkle path;
    out_commitment[j] is output j's commitment;
    in_amount0 + in_amount1 + public_amount = out_amount0 + out_amount1 (mod r), every amount range-checked to 64 bits;
  and recipient is bound by recipient^2 = recipient_sq.
A deposit has two zero-value inputs, a private transfer public_amount 0, a withdrawal public_amount = r - withdrawn.

Variable layout (index -> meaning), P = 4*n_rounds, a level block is the withdraw statement's 2P + 4 variables:
  0 ONE
  1 root | 2 public_amount | 3 token | 4 recipient | 5 nf[0] | 6 nf[1] | 7 out_cm[0] | 8 out_cm[1]      (public, n_pub = 8)
  9 recipient_sq | 10 nf_diff_inv
  11..  input block 0, input block 1; each 68 + 8P + depth*(2P + 4) variables:
        +0 spend_key | +1 blinding | +2 amount | +3..+66 amount bits, LSB first
        +67 owner permutation (P; the owner P = 3 + s + hash(s, 3) is a linear combination, not a variable)
        +67+P commitment: 4 permutations (4P), then cm_out
        +68+5P depth levels
        +68+5P+depth*(2P+4) nullifier: 3 permutations (3P; its output is nf[i] itself)
  then  output block 0, output block 1; each 68 + 4P variables:
        +0 owner | +1 blinding | +2 amount | +3..+66 amount bits | +67 commitment (4P) | +67+4P cm_out
Constraint order:
  recipient^2;
  per input: owner permutation; the commitment's four permutations, r4 * ONE = cm_out; the depth levels exactly as withdraw;
             (root - node_depth) * amount = 0; 64 rows bit*(bit - ONE) = 0, (sum 2^k bit_k - amount) * ONE = 0; the nullifier's
             three permutations, r3 * ONE = nf[i];
  per output: the 65 range rows, the commitment's four permutations and its cm_out row, (cm_out - out_cm[j]) * ONE = 0;
  (in_amount0 + in_amount1 + public_amount - out_amount0 - out_amount1) * ONE = 0;
  (nf[0] - nf[1]) * nf_diff_inv = ONE.
Sizes: n_vars = 283 + 24P + depth*(4P + 8), n_constraints = 273 + 24P + depth*(4P + 6); with 91 rounds at depth 32 that is
55 867 variables and 55 793 constraints, domain 2^16.  The transfer statement has n_pub 8 too and 6P = 2 184 fewer variables,
which no difference of depths (1 464 variables a level) makes up, so a key's shape names its statement.

Note delivery (oracle/notes.py's scheme): the record of an owned note is the record of its four words (P, blinding, token,
amount), and its commitment is the key-4 one.  A wallet with view key v and spending key s scans with (v, P): a record is
owned only if it decrypts under v to an amount below 2^64, its first word is P and the key-4 commitment matches.  Without the
owner check a sender could deliver to v a note owned by another spend key, which the wallet would count but could not spend.
"""
from . import notes
from .bn254 import R
from .mimc7 import N_ROUNDS, multi_hash
from .withdraw_circuit import R1CS, _hash2_witness, _perm_constraints, _perm_witness, lc_add

N_PUB = 8
AMOUNT_BITS = 64
OWNER_KEY, COMMITMENT_KEY, NULLIFIER_KEY = 3, 4, 5
V_ONE, V_ROOT, V_PUB_AMOUNT, V_TOKEN, V_RECIP = range(5)
V_NF = (5, 6)
V_OUT_CM = (7, 8)
V_RSQ, V_NF_INV = 9, 10
V_IN_BASE = 11


def spend_public_key(s, n_rounds: int = N_ROUNDS) -> int:
    return multi_hash([s % R], OWNER_KEY, n_rounds)


def commitment(owner, blinding, token, amount, n_rounds: int = N_ROUNDS) -> int:
    return multi_hash([owner % R, blinding % R, token % R, amount % R], COMMITMENT_KEY, n_rounds)


def nullifier(s, cm, index, n_rounds: int = N_ROUNDS) -> int:
    return multi_hash([s % R, cm % R, index % R], NULLIFIER_KEY, n_rounds)


class Layout:
    def __init__(self, depth: int, n_rounds: int = N_ROUNDS):
        self.depth, self.n_rounds = depth, n_rounds
        P = self.perm = 4 * n_rounds
        self.lvl_size = 2 * P + 4
        self.in_size = 68 + 8 * P + depth * self.lvl_size
        self.out_size = 68 + 4 * P
        self.out_base = V_IN_BASE + 2 * self.in_size
        self.n_vars = self.out_base + 2 * self.out_size
        self.n_constraints = 273 + 24 * P + depth * (4 * P + 6)
        assert self.n_vars == 283 + 24 * P + depth * (4 * P + 8)
        if n_rounds == N_ROUNDS:
            assert (self.n_vars, self.n_constraints) == (9019 + 1464 * depth, 9009 + 1462 * depth)
        # named rows, for the soundness tests
        in_rows = 8 * P + 68 + depth * (2 * P + 3)
        self.row_root = [1 + i * in_rows + 5 * P + 1 + depth * (2 * P + 3) for i in range(2)]
        self.row_nf = [1 + (i + 1) * in_rows - 1 for i in range(2)]
        out_rows = 4 * P + 67
        self.row_out_cm = [1 + 2 * in_rows + (j + 1) * out_rows - 1 for j in range(2)]
        self.row_out_range = [1 + 2 * in_rows + j * out_rows + 64 for j in range(2)]
        self.row_in_range = [r + 65 for r in self.row_root]
        self.row_balance = self.n_constraints - 2
        self.row_nf_diff = self.n_constraints - 1

    def note(self, base):
        """Variables of the note block at `base` (input or output): the parts both kinds share."""
        return dict(key=base, blinding=base + 1, amount=base + 2, bits=base + 3)

    def inp(self, i):
        b = V_IN_BASE + i * self.in_size
        P = self.perm
        v = self.note(b)
        v.update(owner_perm=b + 67, cm=b + 67 + P, cm_out=b + 67 + 5 * P, lvl_base=b + 68 + 5 * P,
                 nf_perm=b + 68 + 5 * P + self.depth * self.lvl_size)
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
    Returns the LC of the result (the caller binds it to a variable, or uses it as a linear combination)."""
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


def _commitment_constraints(cs, owner_lc, v, P, n_rounds):
    xs = [owner_lc, {v["blinding"]: 1}, {V_TOKEN: 1}, {v["amount"]: 1}]
    r4 = _multi_hash_constraints(cs, xs, {V_ONE: COMMITMENT_KEY}, [v["cm"] + k * P for k in range(4)], n_rounds)
    cs.add(r4, {V_ONE: 1}, {v["cm_out"]: 1})


def build_r1cs(depth: int, n_rounds: int = N_ROUNDS) -> R1CS:
    assert 1 <= depth <= 32
    L = Layout(depth, n_rounds)
    P = L.perm
    cs = R1CS(L.n_vars, N_PUB)
    cs.add({V_RECIP: 1}, {V_RECIP: 1}, {V_RSQ: 1})
    for i in range(2):
        v = L.inp(i)
        s = {v["key"]: 1}
        owner = _multi_hash_constraints(cs, [s], {V_ONE: OWNER_KEY}, [v["owner_perm"]], n_rounds)
        _commitment_constraints(cs, owner, v, P, n_rounds)
        cur = v["cm_out"]
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
        _range_constraints(cs, v)
        nf = _multi_hash_constraints(cs, [s, {v["cm_out"]: 1}, index], {V_ONE: NULLIFIER_KEY},
                                     [v["nf_perm"] + k * P for k in range(3)], n_rounds)
        cs.add(nf, {V_ONE: 1}, {V_NF[i]: 1})
    for j in range(2):
        v = L.out(j)
        _range_constraints(cs, v)
        _commitment_constraints(cs, {v["key"]: 1}, v, P, n_rounds)
        cs.add(lc_add({v["cm_out"]: 1}, {V_OUT_CM[j]: R - 1}), {V_ONE: 1}, {})
    i0, i1, o0, o1 = L.inp(0)["amount"], L.inp(1)["amount"], L.out(0)["amount"], L.out(1)["amount"]
    cs.add(lc_add({i0: 1}, {i1: 1}, {V_PUB_AMOUNT: 1}, {o0: R - 1}, {o1: R - 1}), {V_ONE: 1}, {})
    cs.add({V_NF[0]: 1, V_NF[1]: R - 1}, {V_NF_INV: 1}, {V_ONE: 1})
    assert cs.n_constraints == L.n_constraints
    return cs


def _multi_hash_witness(w, xs, key, base, P, n_rounds):
    r = key
    for k, x in enumerate(xs):
        r = (r + x + _perm_witness(w, x, r, base + k * P, n_rounds)) % R
    return r


def _note_witness(w, v, first, owner, blinding, token, amount, P, n_rounds):
    """Fills a note block's first variable (the spend key of an input, the owner of an output), blinding, amount, its low 64
    bits and the commitment of (owner, blinding, token, amount); returns the commitment."""
    w[v["key"]], w[v["blinding"]], w[v["amount"]] = first % R, blinding % R, amount
    for k in range(AMOUNT_BITS):
        w[v["bits"] + k] = (amount >> k) & 1
    w[v["cm_out"]] = _multi_hash_witness(w, [owner % R, w[v["blinding"]], token, amount], COMMITMENT_KEY, v["cm"], P, n_rounds)
    return w[v["cm_out"]]


def witness(root, token, recipient, inputs, outputs, n_rounds: int = N_ROUNDS):
    """Full assignment (list of n_vars ints).
    inputs: two (spend_key, blinding, amount, siblings[depth], path_bits); outputs: two (owner, blinding, amount).
    root is the caller's; public_amount, the nullifiers and the output commitments are derived.  A wrong spend key or any
    other input of nonzero value that does not reach root, or two inputs with one nullifier, give an assignment that does
    not satisfy the R1CS."""
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
    for i, (s, blinding, amount, sibs, bits) in enumerate(inputs):
        assert len(sibs) == depth
        v = L.inp(i)
        s %= R
        owner = _multi_hash_witness(w, [s], OWNER_KEY, v["owner_perm"], P, n_rounds)
        cm = cur = _note_witness(w, v, s, owner, blinding, w[V_TOKEN], amount, P, n_rounds)
        for l in range(depth):
            lv = L.level(i, l)
            sib, bit = sibs[l] % R, (bits >> l) & 1
            left, right = (sib, cur) if bit else (cur, sib)
            w[lv["sib"]], w[lv["bit"]], w[lv["left"]] = sib, bit, left
            cur = _hash2_witness(w, left, right, lv["perm1"], lv["perm2"], lv["out"], n_rounds)
        index = bits & ((1 << depth) - 1)
        w[V_NF[i]] = _multi_hash_witness(w, [s, cm, index], NULLIFIER_KEY, v["nf_perm"], P, n_rounds)
    for j, (owner, blinding, amount) in enumerate(outputs):
        w[V_OUT_CM[j]] = _note_witness(w, L.out(j), owner, owner, blinding, w[V_TOKEN], amount, P, n_rounds)
    a_in = inputs[0][2] + inputs[1][2]
    a_out = outputs[0][2] + outputs[1][2]
    w[V_PUB_AMOUNT] = (a_out - a_in) % R
    d = (w[V_NF[0]] - w[V_NF[1]]) % R
    w[V_NF_INV] = pow(d, R - 2, R) if d else 0
    return w


def encrypt_note(pk, note, e):
    """-> (status, record, commitment) of an owned note (owner, blinding, token, amount) to the view address pk: the record
    notes.encrypt makes of the same four words, the key-4 commitment."""
    st, rec, _ = notes.encrypt(pk, note, e)
    return st, rec, (commitment(*note) if st == notes.ENC_OK else 0)


def scan_notes(view_keys, spend_public_keys, records, commitments):
    """-> (owners, plaintexts) as notes.scan, key j being (view_keys[j], spend_public_keys[j]) and owning a record only if
    the decrypted note's owner is spend_public_keys[j] and its key-4 commitment matches."""
    owners, plain = [], []
    for rec, cm in zip(records, commitments):
        p = notes.prepare(rec, cm)
        owner, note = (notes.MALFORMED, None) if p is None else (notes.NOT_OWNED, None)
        if p is not None:
            Ep, cs = p
            for j, (v, P) in enumerate(zip(view_keys, spend_public_keys)):
                k = notes._key(notes.mul(Ep, v))
                m = [(c - notes._pad(i, k)) % R for i, c in enumerate(cs)]
                if m[3] < 1 << 64 and m[0] == P and commitment(*m) == cm:
                    owner, note = j, tuple(m)
                    break
        owners.append(owner)
        plain.append(bytes(notes.PLAINTEXT_BYTES) if note is None else b"".join(x.to_bytes(32, "little") for x in note))
    return owners, plain
