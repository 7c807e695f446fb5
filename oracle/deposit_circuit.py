"""The frozen privacy-pool *deposit* statement as an R1CS, plus its witness map.

The second statement of the library (DESIGN.md section 3); the product's C++ builder
(owshen_b200/csrc/withdraw_circuit.hpp: DepositBuilder) must reproduce it entry for entry.

Statement (public: commitment, depositor):
  I know (nullifier, secret) such that
    commitment = MultiMiMC7([nullifier, secret], key=0)
  and depositor is bound by depositor^2 = depositor_sq.
The commitment block is the withdraw statement's, so a deposited commitment is a leaf that the withdraw
statement can open.  Amount and token are absent because the withdraw statement has neither.

Variable layout (index -> meaning), PERM = 4*n_rounds:
  0 ONE | 1 commitment | 2 depositor                     (public, n_pub = 2)
  3 nullifier | 4 secret | 5 depositor_sq
  6 ..  commitment block  perm1[PERM] perm2[PERM] out
Constraint order: depositor^2; commitment perm1, perm2, output; (out - commitment) * ONE = 0.
With 91 rounds: 735 variables, 731 constraints, domain 2^10.
"""
from .bn254 import R
from .mimc7 import N_ROUNDS
from .withdraw_circuit import R1CS, _hash2_constraints, _hash2_witness, lc_add

N_PUB = 2
V_ONE, V_CM, V_DEP, V_NULL, V_SECRET, V_DSQ = range(6)
V_CM_BLOCK = 6


class Layout:
    def __init__(self, n_rounds: int = N_ROUNDS):
        self.n_rounds = n_rounds
        self.perm = 4 * n_rounds
        self.cm_base = V_CM_BLOCK
        self.cm_out = self.cm_base + 2 * self.perm
        self.n_vars = self.cm_out + 1
        self.n_constraints = 1 + (2 * self.perm + 1) + 1


def build_r1cs(n_rounds: int = N_ROUNDS) -> R1CS:
    L = Layout(n_rounds)
    cs = R1CS(L.n_vars, N_PUB)
    cs.add({V_DEP: 1}, {V_DEP: 1}, {V_DSQ: 1})
    _hash2_constraints(cs, {V_NULL: 1}, {V_SECRET: 1}, L.cm_base, L.cm_base + L.perm, L.cm_out, n_rounds)
    cs.add(lc_add({L.cm_out: 1}, {V_CM: R - 1}), {V_ONE: 1}, {})
    assert cs.n_constraints == L.n_constraints
    return cs


def witness(nullifier, secret, depositor, n_rounds: int = N_ROUNDS):
    """Full assignment (list of n_vars ints).  The commitment is derived."""
    L = Layout(n_rounds)
    w = [0] * L.n_vars
    w[V_ONE] = 1
    w[V_DEP] = depositor % R
    w[V_NULL] = nullifier % R
    w[V_SECRET] = secret % R
    w[V_DSQ] = w[V_DEP] * w[V_DEP] % R
    w[V_CM] = _hash2_witness(w, w[V_NULL], w[V_SECRET], L.cm_base, L.cm_base + L.perm, L.cm_out, n_rounds)
    return w
