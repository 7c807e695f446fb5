// owshen_b200/csrc/withdraw_circuit.hpp -- host-side builders of the withdraw, deposit, transfer, association, exclusion,
// labeled and labeled association withdraw statements' R1CS (DESIGN.md section 3).  The reference defines no circuit (SURVEY.md
// section 0/8c); these are the product's own definitions, checked entry for entry against the independently written
// oracle/*_circuit.py specs through the og_<statement>_r1cs_export entry points (statement_r1cs below).
//
// withdraw
//   public : root, nullifier_hash, recipient
//   private: nullifier, secret, siblings[depth], bits[depth]
//   nullifier_hash = MultiMiMC7([nullifier], key 1); commitment = MultiMiMC7([nullifier, secret], 0);
//   root = Merkle root from commitment with node = MultiMiMC7([left, right], 0); recipient^2 bound.
// deposit
//   public : commitment, depositor
//   private: nullifier, secret
//   commitment = MultiMiMC7([nullifier, secret], 0) (the withdraw statement's leaf); depositor^2 bound.
// transfer
//   public : root, public_amount, token, recipient, nullifier_hash[2], out_commitment[2]
//   private: two input notes (nullifier, secret, amount, siblings[depth], bits[depth]), two output notes
//   note commitment = MultiMiMC7([nullifier, secret, token, amount], 0), amounts range-checked to 64 bits;
//   nonzero inputs open under root; in0 + in1 + public_amount = out0 + out1; nh[0] != nh[1]; recipient^2 bound.
// association
//   public : root, nullifier_hash, recipient, association_root
//   private: nullifier, secret, siblings[depth], bits[depth], assoc_siblings[depth], assoc_bits[depth]
//   withdraw's nullifier hash and commitment; the commitment reaches root along the pool path and association_root along
//   the association path (one depth for both trees); recipient^2 bound.
// exclusion
//   public : root, nullifier_hash, recipient, exclusion_root
//   private: nullifier, secret, siblings[depth], bits[depth], low, next, excl_siblings[depth], excl_bits[depth]
//   withdraw's nullifier hash, commitment and pool path; with x = ONE + sum 2^l bits[l] (leaf index + 1), low, next,
//   x - low - 1 and next - x - 1 range-checked to 33 bits, and MultiMiMC7([low, next], 0) reaching exclusion_root along the
//   exclusion path (one depth for both trees); recipient^2 bound.
// labeled
//   public : root, nullifier_hash, recipient, exclusion_root, token, withdrawn, change_commitment
//   private: nullifier, secret, amount, label, siblings[depth], bits[depth], change_nullifier, change_secret, low, next,
//            excl_siblings[depth], excl_bits[depth]
//   withdraw's nullifier hash; precommitment = MultiMiMC7([nullifier, secret], 2), leaf = MultiMiMC7([pre, token, amount,
//   label], 2) reaching root along the pool path; amount, withdrawn, change = amount - withdrawn range-checked to 64 bits and
//   label to 32; change_commitment = the leaf of (change_nullifier, change_secret, token, change, label); the exclusion
//   statement's bracket on x = label + 1 and its blocklist path to exclusion_root; recipient^2 bound.
// labeled_association
//   public : root, nullifier_hash, recipient, association_root, token, withdrawn, change_commitment
//   private: nullifier, secret, amount, label, siblings[depth], bits[depth], change_nullifier, change_secret,
//            assoc_siblings[depth], assoc_bits[depth]
//   the labeled statement's note part (LabeledNoteBuilder); assoc_leaf = label + 1 reaching association_root along the
//   association path (one depth for both trees); recipient^2 bound.
// owned_transfer
//   public : root, public_amount, token, recipient, nullifier[2], out_commitment[2]
//   private: two input notes (spend_key, blinding, amount, siblings[depth], bits[depth]), two output notes (owner, blinding,
//            amount)
//   owner = MultiMiMC7([spend_key], 3); note commitment = MultiMiMC7([owner, blinding, token, amount], 4); nullifier =
//   MultiMiMC7([spend_key, commitment, leaf index], 5); otherwise the transfer statement's rows.
// owned_labeled_transfer
//   public : root, association_root, token, withdrawn, recipient, nullifier[2], out_commitment[2]
//   private: label, two input notes (spend_key, blinding, amount, siblings[depth], bits[depth]), two output notes (owner,
//            blinding, amount), assoc_siblings[depth], assoc_bits[depth]
//   owner = MultiMiMC7([spend_key], 3); precommitment = MultiMiMC7([owner, blinding], 6); leaf = MultiMiMC7([pre, token,
//   amount, label], 7) with one label for all four notes; nullifier = MultiMiMC7([spend_key, leaf, leaf index], 5); label
//   range-checked to 32 bits, withdrawn and the amounts to 64; in0 + in1 = out0 + out1 + withdrawn; nonzero inputs open
//   under root; nf[0] != nf[1]; assoc_leaf = label + 1 reaching association_root; recipient^2 bound.
// ragequit
//   public : root, token, amount, label, recipient, nullifier
//   private: spend_key, blinding, siblings[depth], bits[depth]
//   the owned labeled transfer's owner, precommitment, leaf and nullifier for one note, spent whole; the leaf reaches root
//   unconditionally; no range rows (the leaf binds amount and label, and every key-7 leaf in the pool was range-checked on
//   its way in); no association path; recipient^2 bound.
#pragma once
#include <map>
#include <vector>
#include "host_math.hpp"
#include "mimc.cuh"

namespace og {

typedef std::map<uint32_t, Fr> LC;   // variable -> coefficient (Montgomery), zero terms erased, sorted by variable

inline void lc_add_term(LC& lc, uint32_t var, const Fr& coeff) {
    auto it = lc.find(var);
    if (it == lc.end()) { if (!coeff.is_zero()) lc[var] = coeff; return; }
    Fr s = it->second + coeff;
    if (s.is_zero()) lc.erase(it); else it->second = s;
}
inline LC lc_sum(std::initializer_list<const LC*> parts) {
    LC out;
    for (const LC* p : parts) for (auto& kv : *p) lc_add_term(out, kv.first, kv.second);
    return out;
}
inline LC lc_var(uint32_t v) { LC l; l[v] = Fr::one(); return l; }
inline LC lc_neg_var(uint32_t v) { LC l; l[v] = Fr::one().neg(); return l; }

struct Csr {
    std::vector<uint32_t> row_ptr{0}, col;
    std::vector<Fr> val;
    void push_row(const LC& lc) {
        for (auto& kv : lc) { col.push_back(kv.first); val.push_back(kv.second); }
        row_ptr.push_back((uint32_t)col.size());
    }
    uint32_t rows() const { return (uint32_t)row_ptr.size() - 1; }
};

struct R1cs {
    uint32_t n_vars = 0, n_pub = 0;
    Csr A, B, C;
    void add(const LC& a, const LC& b, const LC& c) { A.push_row(a); B.push_row(b); C.push_row(c); }
    uint32_t n_constraints() const { return A.rows(); }
};

// the MiMC7, Merkle-path and range gadgets the statements are made of
struct Mimc7Builder {
    R1cs cs;
    Fr consts[MIMC_ROUNDS];
    uint32_t n_rounds;

    explicit Mimc7Builder(uint32_t rounds) : n_rounds(rounds) { mimc7_round_constants(consts); }

    // MiMC7 permutation rounds over x with key k; returns the LC of hash(x, k) = perm + k
    LC perm(const LC& x, const LC& k, uint32_t base) {
        LC prev = x;
        for (uint32_t i = 0; i < n_rounds; i++) {
            uint32_t t2 = base + 4 * i, t4 = t2 + 1, t6 = t2 + 2, t7 = t2 + 3;
            LC c; if (!consts[i].is_zero()) c[0] = consts[i];
            LC t = lc_sum({&prev, &k, &c});
            cs.add(t, t, lc_var(t2));
            cs.add(lc_var(t2), lc_var(t2), lc_var(t4));
            cs.add(lc_var(t4), lc_var(t2), lc_var(t6));
            cs.add(lc_var(t6), t, lc_var(t7));
            prev = lc_var(t7);
        }
        return lc_sum({&prev, &k});
    }
    // MultiMiMC7(xs, key): r = key; r = r + x + hash(x, r) per input, the i-th permutation's rounds at bases[i];
    // then r * ONE = out
    void multi_hash(std::initializer_list<const LC*> xs, const LC& key, std::initializer_list<uint32_t> bases, uint32_t out) {
        LC r = key;
        const uint32_t* base = bases.begin();
        for (const LC* x : xs) {
            LC h = perm(*x, r, *base++);
            r = lc_sum({&r, x, &h});
        }
        cs.add(r, lc_var(0), lc_var(out));
    }
    void hash2(const LC& left, const LC& right, uint32_t perm1, uint32_t perm2, uint32_t out) {
        multi_hash({&left, &right}, LC(), {perm1, perm2}, out);
    }
    // The `depth` levels of a Merkle path from the leaf variable `cur`, level l's block (sibling, bit, left, perm1, perm2, out)
    // at base + l * lvl_size: bit * (bit - ONE) = 0, bit * (sib - cur) = left - cur, then left, right = sib + cur - left
    // hashed into out.  Returns the variable of the root it reaches.
    uint32_t merkle_path(uint32_t cur, uint32_t base, uint32_t lvl_size, uint32_t depth) {
        const uint32_t P = 4 * n_rounds;
        for (uint32_t l = 0; l < depth; l++) {
            uint32_t lb = base + l * lvl_size;
            uint32_t sib = lb, bit = lb + 1, left = lb + 2, p1 = lb + 3, p2 = lb + 3 + P, out = lb + 3 + 2 * P;
            LC vbit = lc_var(bit), m1 = lc_neg_var(0), vsib = lc_var(sib), ncur = lc_neg_var(cur), vleft = lc_var(left), vcur = lc_var(cur);
            LC nleft = lc_neg_var(left);
            cs.add(vbit, lc_sum({&vbit, &m1}), LC());
            cs.add(vbit, lc_sum({&vsib, &ncur}), lc_sum({&vleft, &ncur}));
            LC right = lc_sum({&vsib, &vcur, &nleft});
            hash2(vleft, right, p1, p2, out);
            cur = out;
        }
        return cur;
    }
    // n_bits range rows: bit_k * (bit_k - ONE) = 0 for the variables bits + k, then (sum 2^k bit_k - value) * ONE = 0
    void range(const LC& value, uint32_t bits, uint32_t n_bits) {
        LC m1 = lc_neg_var(0), packed;
        for (auto& kv : value) lc_add_term(packed, kv.first, kv.second.neg());
        Fr pow2 = Fr::one();
        for (uint32_t k = 0; k < n_bits; k++) {
            LC vbit = lc_var(bits + k);
            cs.add(vbit, lc_sum({&vbit, &m1}), LC());
            lc_add_term(packed, bits + k, pow2);
            pow2 = pow2 + pow2;
        }
        cs.add(packed, lc_var(0), LC());
    }
};

struct WithdrawBuilder {
    static R1cs build(uint32_t depth, uint32_t n_rounds = MIMC_ROUNDS) {
        Mimc7Builder b(n_rounds);
        WithdrawLayout L = WithdrawLayout::make(depth, n_rounds);
        b.cs.n_vars = L.n_vars;
        b.cs.n_pub = WITHDRAW_N_PUB;
        const uint32_t V_ONE = 0, V_ROOT = 1, V_NHASH = 2, V_RECIP = 3, V_NULL = 4, V_SECRET = 5, V_RSQ = 6, V_NH_PERM = 7;
        b.cs.add(lc_var(V_RECIP), lc_var(V_RECIP), lc_var(V_RSQ));
        LC nu = lc_var(V_NULL);
        b.multi_hash({&nu}, lc_var(V_ONE), {V_NH_PERM}, V_NHASH);
        b.hash2(lc_var(V_NULL), lc_var(V_SECRET), L.cm_base, L.cm_base + L.perm, L.cm_out);
        const uint32_t cur = b.merkle_path(L.cm_out, L.lvl_base, L.lvl_size, depth);
        LC vcur = lc_var(cur), nroot = lc_neg_var(V_ROOT);
        b.cs.add(lc_sum({&vcur, &nroot}), lc_var(V_ONE), LC());
        return b.cs;
    }
};

struct DepositBuilder {
    static R1cs build(uint32_t n_rounds = MIMC_ROUNDS) {
        Mimc7Builder b(n_rounds);
        DepositLayout L = DepositLayout::make(n_rounds);
        b.cs.n_vars = L.n_vars;
        b.cs.n_pub = DEPOSIT_N_PUB;
        const uint32_t V_ONE = 0, V_CM = 1, V_DEP = 2, V_NULL = 3, V_SECRET = 4, V_DSQ = 5;
        b.cs.add(lc_var(V_DEP), lc_var(V_DEP), lc_var(V_DSQ));
        b.hash2(lc_var(V_NULL), lc_var(V_SECRET), L.cm_base, L.cm_base + L.perm, L.cm_out);
        LC vout = lc_var(L.cm_out), ncm = lc_neg_var(V_CM);
        b.cs.add(lc_sum({&vout, &ncm}), lc_var(V_ONE), LC());
        return b.cs;
    }
};

struct TransferBuilder {
    // commitment = MultiMiMC7([nullifier, secret, token, amount], 0) of the note block at `v`, rounds from `cm`
    static void commitment(Mimc7Builder& b, uint32_t v, uint32_t cm, uint32_t cm_out, uint32_t P) {
        LC nu = lc_var(v), se = lc_var(v + 1), tok = lc_var(3), am = lc_var(v + 2);
        b.multi_hash({&nu, &se, &tok, &am}, LC(), {cm, cm + P, cm + 2 * P, cm + 3 * P}, cm_out);
    }

    static R1cs build(uint32_t depth, uint32_t n_rounds = MIMC_ROUNDS) {
        Mimc7Builder b(n_rounds);
        TransferLayout L = TransferLayout::make(depth, n_rounds);
        b.cs.n_vars = L.n_vars;
        b.cs.n_pub = TRANSFER_N_PUB;
        const uint32_t V_ONE = 0, V_ROOT = 1, V_PUB_AMOUNT = 2, V_RECIP = 4, V_NH = 5, V_OUT_CM = 7, V_RSQ = 9, V_NH_INV = 10;
        const uint32_t P = L.perm;
        b.cs.add(lc_var(V_RECIP), lc_var(V_RECIP), lc_var(V_RSQ));
        for (uint32_t i = 0; i < 2; i++) {
            const uint32_t v = L.inp(i);
            LC nu = lc_var(v);
            b.multi_hash({&nu}, lc_var(V_ONE), {v + L.nh_perm}, V_NH + i);
            b.range(lc_var(v + 2), v + 3, TRANSFER_AMOUNT_BITS);
            commitment(b, v, v + L.in_cm, v + L.in_cm_out, P);
            const uint32_t cur = b.merkle_path(v + L.in_cm_out, v + L.lvl_base, L.lvl_size, depth);
            LC vroot = lc_var(V_ROOT), ncur = lc_neg_var(cur);
            b.cs.add(lc_sum({&vroot, &ncur}), lc_var(v + 2), LC());
        }
        for (uint32_t j = 0; j < 2; j++) {
            const uint32_t v = L.out(j);
            b.range(lc_var(v + 2), v + 3, TRANSFER_AMOUNT_BITS);
            commitment(b, v, v + L.out_cm, v + L.out_cm_out, P);
            LC vout = lc_var(v + L.out_cm_out), ncm = lc_neg_var(V_OUT_CM + j);
            b.cs.add(lc_sum({&vout, &ncm}), lc_var(V_ONE), LC());
        }
        LC i0 = lc_var(L.inp(0) + 2), i1 = lc_var(L.inp(1) + 2), pa = lc_var(V_PUB_AMOUNT);
        LC o0 = lc_neg_var(L.out(0) + 2), o1 = lc_neg_var(L.out(1) + 2);
        b.cs.add(lc_sum({&i0, &i1, &pa, &o0, &o1}), lc_var(V_ONE), LC());
        LC nh0 = lc_var(V_NH), nh1 = lc_neg_var(V_NH + 1);
        b.cs.add(lc_sum({&nh0, &nh1}), lc_var(V_NH_INV), lc_var(V_ONE));
        return b.cs;
    }
};

struct AssociationBuilder {
    static R1cs build(uint32_t depth, uint32_t n_rounds = MIMC_ROUNDS) {
        Mimc7Builder b(n_rounds);
        AssociationLayout L = AssociationLayout::make(depth, n_rounds);
        b.cs.n_vars = L.n_vars;
        b.cs.n_pub = ASSOCIATION_N_PUB;
        const uint32_t V_ONE = 0, V_ROOT = 1, V_NHASH = 2, V_RECIP = 3, V_AROOT = 4, V_NULL = 5, V_SECRET = 6, V_RSQ = 7, V_NH_PERM = 8;
        b.cs.add(lc_var(V_RECIP), lc_var(V_RECIP), lc_var(V_RSQ));
        LC nu = lc_var(V_NULL);
        b.multi_hash({&nu}, lc_var(V_ONE), {V_NH_PERM}, V_NHASH);
        b.hash2(lc_var(V_NULL), lc_var(V_SECRET), L.cm_base, L.cm_base + L.perm, L.cm_out);
        const uint32_t bases[2] = {L.pool_base, L.assoc_base}, roots[2] = {V_ROOT, V_AROOT};
        for (int t = 0; t < 2; t++) {
            const uint32_t cur = b.merkle_path(L.cm_out, bases[t], L.lvl_size, depth);
            LC vcur = lc_var(cur), nroot = lc_neg_var(roots[t]);
            b.cs.add(lc_sum({&vcur, &nroot}), lc_var(V_ONE), LC());
        }
        return b.cs;
    }
};

struct ExclusionBuilder {
    static R1cs build(uint32_t depth, uint32_t n_rounds = MIMC_ROUNDS) {
        Mimc7Builder b(n_rounds);
        ExclusionLayout L = ExclusionLayout::make(depth, n_rounds);
        b.cs.n_vars = L.n_vars;
        b.cs.n_pub = EXCLUSION_N_PUB;
        const uint32_t V_ONE = 0, V_ROOT = 1, V_NHASH = 2, V_RECIP = 3, V_XROOT = 4, V_NULL = 5, V_SECRET = 6, V_RSQ = 7, V_LOW = 8,
                       V_NEXT = 9, V_NH_PERM = 10;
        b.cs.add(lc_var(V_RECIP), lc_var(V_RECIP), lc_var(V_RSQ));
        LC nu = lc_var(V_NULL);
        b.multi_hash({&nu}, lc_var(V_ONE), {V_NH_PERM}, V_NHASH);
        b.hash2(lc_var(V_NULL), lc_var(V_SECRET), L.cm_base, L.cm_base + L.perm, L.cm_out);
        const uint32_t pool_root = b.merkle_path(L.cm_out, L.pool_base, L.lvl_size, depth);
        LC vpool = lc_var(pool_root), nroot = lc_neg_var(V_ROOT);
        b.cs.add(lc_sum({&vpool, &nroot}), lc_var(V_ONE), LC());
        // x = ONE + sum 2^l bit_l over the pool levels' bits: the note's leaf index + 1, its key in the blocklist tree
        LC x = lc_var(V_ONE), nx;
        Fr pow2 = Fr::one();
        for (uint32_t l = 0; l < depth; l++) {
            lc_add_term(x, L.pool_base + l * L.lvl_size + 1, pow2);
            pow2 = pow2 + pow2;
        }
        for (auto& kv : x) lc_add_term(nx, kv.first, kv.second.neg());
        LC low = lc_var(V_LOW), next = lc_var(V_NEXT), nlow = lc_neg_var(V_LOW), m1 = lc_neg_var(V_ONE);
        b.range(low, L.low_bits, EXCLUSION_RANGE_BITS);
        b.range(next, L.next_bits, EXCLUSION_RANGE_BITS);
        b.range(lc_sum({&x, &nlow, &m1}), L.gap_lo_bits, EXCLUSION_RANGE_BITS);      // x - low - 1
        b.range(lc_sum({&next, &nx, &m1}), L.gap_hi_bits, EXCLUSION_RANGE_BITS);     // next - x - 1
        b.hash2(low, next, L.leaf_base, L.leaf_base + L.perm, L.leaf_out);
        const uint32_t excl_root = b.merkle_path(L.leaf_out, L.excl_base, L.lvl_size, depth);
        LC vexcl = lc_var(excl_root), nxroot = lc_neg_var(V_XROOT);
        b.cs.add(lc_sum({&vexcl, &nxroot}), lc_var(V_ONE), LC());
        return b.cs;
    }
};

// The note part of the labeled and labeled association statements, whose layouts share variables 0..14 (variable 4 is the
// exclusion or association root) and the names of their note blocks; the nullifier-hash permutation sits just below the
// precommitment block.
struct LabeledNoteBuilder {
    static constexpr uint32_t V_ONE = 0, V_ROOT = 1, V_NHASH = 2, V_RECIP = 3, V_TOKEN = 5, V_WITHDRAWN = 6, V_CHANGE_CM = 7,
                              V_NULL = 8, V_SECRET = 9, V_RSQ = 10, V_AMOUNT = 11, V_LABEL = 12, V_CNULL = 13, V_CSECRET = 14;
    static LC key() { LC k; k[V_ONE] = Fr::from_u32(LABELED_KEY); return k; }
    static LC change() { LC am = lc_var(V_AMOUNT), nwd = lc_neg_var(V_WITHDRAWN); return lc_sum({&am, &nwd}); }   // amount - withdrawn

    // recipient; the nullifier hash; the precommitment and the leaf, the pool levels and the pool root row; the amount,
    // withdrawn, change and label ranges
    template <class Layout> static void spend(Mimc7Builder& b, const Layout& L) {
        // the base lists take copies: host GCC rejects the dependent member accesses inside these braced lists
        const uint32_t P = L.perm, pre_base = L.pre_base, leaf_base = L.leaf_base;
        const LC k = key();
        b.cs.add(lc_var(V_RECIP), lc_var(V_RECIP), lc_var(V_RSQ));
        LC nu = lc_var(V_NULL), se = lc_var(V_SECRET), tok = lc_var(V_TOKEN), am = lc_var(V_AMOUNT), la = lc_var(V_LABEL);
        b.multi_hash({&nu}, lc_var(V_ONE), {pre_base - P}, V_NHASH);
        b.multi_hash({&nu, &se}, k, {pre_base, pre_base + P}, L.pre_out);
        LC pre = lc_var(L.pre_out);
        b.multi_hash({&pre, &tok, &am, &la}, k, {leaf_base, leaf_base + P, leaf_base + 2 * P, leaf_base + 3 * P}, L.leaf_out);
        const uint32_t pool_root = b.merkle_path(L.leaf_out, L.pool_base, L.lvl_size, L.depth);
        LC vpool = lc_var(pool_root), nroot = lc_neg_var(V_ROOT);
        b.cs.add(lc_sum({&vpool, &nroot}), lc_var(V_ONE), LC());
        b.range(am, L.amount_bits, LABELED_AMOUNT_BITS);
        b.range(lc_var(V_WITHDRAWN), L.withdrawn_bits, LABELED_AMOUNT_BITS);
        b.range(change(), L.change_bits, LABELED_AMOUNT_BITS);
        b.range(la, L.label_bits, LABELED_LABEL_BITS);
    }
    // the change precommitment, then the change commitment with its output row bound to change_commitment
    template <class Layout> static void change_note(Mimc7Builder& b, const Layout& L) {
        const uint32_t P = L.perm, cpre_base = L.cpre_base, ccm_base = L.ccm_base;
        const LC k = key(), ch = change();
        LC cnu = lc_var(V_CNULL), cse = lc_var(V_CSECRET), tok = lc_var(V_TOKEN), la = lc_var(V_LABEL);
        b.multi_hash({&cnu, &cse}, k, {cpre_base, cpre_base + P}, L.cpre_out);
        LC cpre = lc_var(L.cpre_out);
        b.multi_hash({&cpre, &tok, &ch, &la}, k, {ccm_base, ccm_base + P, ccm_base + 2 * P, ccm_base + 3 * P}, V_CHANGE_CM);
    }
};

struct LabeledBuilder {
    static R1cs build(uint32_t depth, uint32_t n_rounds = MIMC_ROUNDS) {
        Mimc7Builder b(n_rounds);
        LabeledLayout L = LabeledLayout::make(depth, n_rounds);
        b.cs.n_vars = L.n_vars;
        b.cs.n_pub = LABELED_N_PUB;
        const uint32_t V_ONE = 0, V_XROOT = 4, V_LABEL = 12, V_LOW = 15, V_NEXT = 16;
        LabeledNoteBuilder::spend(b, L);
        // x = label + 1, the deposit's key in the blocklist tree
        LC la = lc_var(V_LABEL), one = lc_var(V_ONE), x = lc_sum({&la, &one}), nx;
        for (auto& kv : x) lc_add_term(nx, kv.first, kv.second.neg());
        LC low = lc_var(V_LOW), next = lc_var(V_NEXT), nlow = lc_neg_var(V_LOW), m1 = lc_neg_var(V_ONE);
        b.range(low, L.low_bits, EXCLUSION_RANGE_BITS);
        b.range(next, L.next_bits, EXCLUSION_RANGE_BITS);
        b.range(lc_sum({&x, &nlow, &m1}), L.gap_lo_bits, EXCLUSION_RANGE_BITS);      // x - low - 1
        b.range(lc_sum({&next, &nx, &m1}), L.gap_hi_bits, EXCLUSION_RANGE_BITS);     // next - x - 1
        LabeledNoteBuilder::change_note(b, L);
        b.hash2(low, next, L.xleaf_base, L.xleaf_base + L.perm, L.xleaf_out);
        const uint32_t excl_root = b.merkle_path(L.xleaf_out, L.excl_base, L.lvl_size, depth);
        LC vexcl = lc_var(excl_root), nxroot = lc_neg_var(V_XROOT);
        b.cs.add(lc_sum({&vexcl, &nxroot}), lc_var(V_ONE), LC());
        return b.cs;
    }
};

struct LabeledAssociationBuilder {
    static R1cs build(uint32_t depth, uint32_t n_rounds = MIMC_ROUNDS) {
        Mimc7Builder b(n_rounds);
        LabeledAssociationLayout L = LabeledAssociationLayout::make(depth, n_rounds);
        b.cs.n_vars = L.n_vars;
        b.cs.n_pub = LABELED_ASSOCIATION_N_PUB;
        const uint32_t V_ONE = 0, V_AROOT = 4, V_LABEL = 12, V_ALEAF = 15;
        LabeledNoteBuilder::spend(b, L);
        LabeledNoteBuilder::change_note(b, L);
        // assoc_leaf = label + 1, the deposit's leaf in the provider's tree of approved labels
        LC la = lc_var(V_LABEL), one = lc_var(V_ONE), nleaf = lc_neg_var(V_ALEAF);
        b.cs.add(lc_sum({&la, &one, &nleaf}), lc_var(V_ONE), LC());
        const uint32_t assoc_root = b.merkle_path(V_ALEAF, L.assoc_base, L.lvl_size, depth);
        LC vassoc = lc_var(assoc_root), naroot = lc_neg_var(V_AROOT);
        b.cs.add(lc_sum({&vassoc, &naroot}), lc_var(V_ONE), LC());
        return b.cs;
    }
};

struct OwnedTransferBuilder {
    // commitment = MultiMiMC7([owner, blinding, token, amount], 4) of the note block at `v`, rounds from `cm`
    static void commitment(Mimc7Builder& b, const LC& owner, uint32_t v, uint32_t cm, uint32_t cm_out, uint32_t P) {
        LC key; key[0] = Fr::from_u32(OWNED_COMMITMENT_KEY);
        LC bl = lc_var(v + 1), tok = lc_var(3), am = lc_var(v + 2);
        b.multi_hash({&owner, &bl, &tok, &am}, key, {cm, cm + P, cm + 2 * P, cm + 3 * P}, cm_out);
    }

    static R1cs build(uint32_t depth, uint32_t n_rounds = MIMC_ROUNDS) {
        Mimc7Builder b(n_rounds);
        OwnedTransferLayout L = OwnedTransferLayout::make(depth, n_rounds);
        b.cs.n_vars = L.n_vars;
        b.cs.n_pub = OWNED_TRANSFER_N_PUB;
        const uint32_t V_ONE = 0, V_ROOT = 1, V_PUB_AMOUNT = 2, V_RECIP = 4, V_NF = 5, V_OUT_CM = 7, V_RSQ = 9, V_NF_INV = 10;
        const uint32_t P = L.perm;
        b.cs.add(lc_var(V_RECIP), lc_var(V_RECIP), lc_var(V_RSQ));
        for (uint32_t i = 0; i < 2; i++) {
            const uint32_t v = L.inp(i);
            // owner P = MultiMiMC7([s], 3) = 3 + s + hash(s, 3), kept as a linear combination
            LC s = lc_var(v), k3; k3[V_ONE] = Fr::from_u32(OWNED_OWNER_KEY);
            LC h = b.perm(s, k3, v + L.owner_perm);
            LC owner = lc_sum({&k3, &s, &h});
            commitment(b, owner, v, v + L.in_cm, v + L.in_cm_out, P);
            const uint32_t cur = b.merkle_path(v + L.in_cm_out, v + L.lvl_base, L.lvl_size, depth);
            LC vroot = lc_var(V_ROOT), ncur = lc_neg_var(cur);
            b.cs.add(lc_sum({&vroot, &ncur}), lc_var(v + 2), LC());
            b.range(lc_var(v + 2), v + 3, TRANSFER_AMOUNT_BITS);
            // nullifier = MultiMiMC7([s, cm, index], 5), index = sum 2^l bit_l over the path bits, bound to nf[i] directly
            LC cm = lc_var(v + L.in_cm_out), index, k5; k5[V_ONE] = Fr::from_u32(OWNED_NULLIFIER_KEY);
            Fr pow2 = Fr::one();
            for (uint32_t l = 0; l < depth; l++) {
                lc_add_term(index, v + L.lvl_base + l * L.lvl_size + 1, pow2);
                pow2 = pow2 + pow2;
            }
            const uint32_t nf = v + L.nf_perm;
            b.multi_hash({&s, &cm, &index}, k5, {nf, nf + P, nf + 2 * P}, V_NF + i);
        }
        for (uint32_t j = 0; j < 2; j++) {
            const uint32_t v = L.out(j);
            b.range(lc_var(v + 2), v + 3, TRANSFER_AMOUNT_BITS);
            commitment(b, lc_var(v), v, v + L.out_cm, v + L.out_cm_out, P);
            LC vout = lc_var(v + L.out_cm_out), ncm = lc_neg_var(V_OUT_CM + j);
            b.cs.add(lc_sum({&vout, &ncm}), lc_var(V_ONE), LC());
        }
        LC i0 = lc_var(L.inp(0) + 2), i1 = lc_var(L.inp(1) + 2), pa = lc_var(V_PUB_AMOUNT);
        LC o0 = lc_neg_var(L.out(0) + 2), o1 = lc_neg_var(L.out(1) + 2);
        b.cs.add(lc_sum({&i0, &i1, &pa, &o0, &o1}), lc_var(V_ONE), LC());
        LC nf0 = lc_var(V_NF), nf1 = lc_neg_var(V_NF + 1);
        b.cs.add(lc_sum({&nf0, &nf1}), lc_var(V_NF_INV), lc_var(V_ONE));
        return b.cs;
    }
};

struct OwnedLabeledTransferBuilder {
    static constexpr uint32_t V_ONE = 0, V_ROOT = 1, V_AROOT = 2, V_TOKEN = 3, V_WITHDRAWN = 4, V_RECIP = 5, V_NF = 6, V_OUT_CM = 8,
                              V_RSQ = 10, V_NF_INV = 11, V_LABEL = 12, V_ALEAF = 13;
    // the precommitment MultiMiMC7([owner, blinding], 6) and the leaf MultiMiMC7([pre, token, amount, label], 7) of the note
    // block at `v`, each with its output row; `n` is the block's precommitment offset (an input's sits P after an output's)
    static void note(Mimc7Builder& b, const OwnedLabeledTransferLayout& L, const LC& owner, uint32_t v, uint32_t n) {
        const uint32_t P = L.perm, pre = v + n + L.pre, leaf = v + n + L.leaf;
        LC k6, k7; k6[V_ONE] = Fr::from_u32(OWNED_LABELED_PRE_KEY); k7[V_ONE] = Fr::from_u32(OWNED_LABELED_LEAF_KEY);
        LC bl = lc_var(v + 1), tok = lc_var(V_TOKEN), am = lc_var(v + 2), la = lc_var(V_LABEL);
        b.multi_hash({&owner, &bl}, k6, {pre, pre + P}, v + n + L.pre_out);
        LC vpre = lc_var(v + n + L.pre_out);
        b.multi_hash({&vpre, &tok, &am, &la}, k7, {leaf, leaf + P, leaf + 2 * P, leaf + 3 * P}, v + n + L.leaf_out);
    }

    static R1cs build(uint32_t depth, uint32_t n_rounds = MIMC_ROUNDS) {
        Mimc7Builder b(n_rounds);
        OwnedLabeledTransferLayout L = OwnedLabeledTransferLayout::make(depth, n_rounds);
        b.cs.n_vars = L.n_vars;
        b.cs.n_pub = OWNED_LABELED_TRANSFER_N_PUB;
        const uint32_t P = L.perm;
        b.cs.add(lc_var(V_RECIP), lc_var(V_RECIP), lc_var(V_RSQ));
        b.range(lc_var(V_LABEL), L.label_bits, LABELED_LABEL_BITS);
        b.range(lc_var(V_WITHDRAWN), L.withdrawn_bits, LABELED_AMOUNT_BITS);
        for (uint32_t i = 0; i < 2; i++) {
            const uint32_t v = L.inp(i);
            // owner P = MultiMiMC7([s], 3) = 3 + s + hash(s, 3), kept as a linear combination
            LC s = lc_var(v), k3; k3[V_ONE] = Fr::from_u32(OWNED_OWNER_KEY);
            LC h = b.perm(s, k3, v + L.owner_perm);
            LC owner = lc_sum({&k3, &s, &h});
            note(b, L, owner, v, P);
            const uint32_t leaf = v + P + L.leaf_out;
            const uint32_t cur = b.merkle_path(leaf, v + L.lvl_base, L.lvl_size, depth);
            LC vroot = lc_var(V_ROOT), ncur = lc_neg_var(cur);
            b.cs.add(lc_sum({&vroot, &ncur}), lc_var(v + 2), LC());
            b.range(lc_var(v + 2), v + 3, LABELED_AMOUNT_BITS);
            // nullifier = MultiMiMC7([s, leaf, index], 5), index = sum 2^l bit_l over the path bits, bound to nf[i] directly
            LC vleaf = lc_var(leaf), index, k5; k5[V_ONE] = Fr::from_u32(OWNED_NULLIFIER_KEY);
            Fr pow2 = Fr::one();
            for (uint32_t l = 0; l < depth; l++) {
                lc_add_term(index, v + L.lvl_base + l * L.lvl_size + 1, pow2);
                pow2 = pow2 + pow2;
            }
            const uint32_t nf = v + L.nf_perm;
            b.multi_hash({&s, &vleaf, &index}, k5, {nf, nf + P, nf + 2 * P}, V_NF + i);
        }
        for (uint32_t j = 0; j < 2; j++) {
            const uint32_t v = L.out(j);
            b.range(lc_var(v + 2), v + 3, LABELED_AMOUNT_BITS);
            note(b, L, lc_var(v), v, 0);
            LC vout = lc_var(v + L.leaf_out), ncm = lc_neg_var(V_OUT_CM + j);
            b.cs.add(lc_sum({&vout, &ncm}), lc_var(V_ONE), LC());
        }
        // in0 + in1 = out0 + out1 + withdrawn: every term is range-checked below 2^64, so it holds over the integers
        LC i0 = lc_var(L.inp(0) + 2), i1 = lc_var(L.inp(1) + 2), nwd = lc_neg_var(V_WITHDRAWN);
        LC o0 = lc_neg_var(L.out(0) + 2), o1 = lc_neg_var(L.out(1) + 2);
        b.cs.add(lc_sum({&i0, &i1, &o0, &o1, &nwd}), lc_var(V_ONE), LC());
        LC nf0 = lc_var(V_NF), nf1 = lc_neg_var(V_NF + 1);
        b.cs.add(lc_sum({&nf0, &nf1}), lc_var(V_NF_INV), lc_var(V_ONE));
        // assoc_leaf = label + 1, the deposit's leaf in the provider's tree of approved labels
        LC la = lc_var(V_LABEL), one = lc_var(V_ONE), nleaf = lc_neg_var(V_ALEAF);
        b.cs.add(lc_sum({&la, &one, &nleaf}), lc_var(V_ONE), LC());
        const uint32_t assoc_root = b.merkle_path(V_ALEAF, L.assoc_base, L.lvl_size, depth);
        LC vassoc = lc_var(assoc_root), naroot = lc_neg_var(V_AROOT);
        b.cs.add(lc_sum({&vassoc, &naroot}), lc_var(V_ONE), LC());
        return b.cs;
    }
};

struct RagequitBuilder {
    static constexpr uint32_t V_ONE = 0, V_ROOT = 1, V_TOKEN = 2, V_AMOUNT = 3, V_LABEL = 4, V_RECIP = 5, V_NF = 6, V_RSQ = 7,
                              V_KEY = 8, V_BLINDING = 9;

    static R1cs build(uint32_t depth, uint32_t n_rounds = MIMC_ROUNDS) {
        Mimc7Builder b(n_rounds);
        RagequitLayout L = RagequitLayout::make(depth, n_rounds);
        b.cs.n_vars = L.n_vars;
        b.cs.n_pub = RAGEQUIT_N_PUB;
        const uint32_t P = L.perm;
        b.cs.add(lc_var(V_RECIP), lc_var(V_RECIP), lc_var(V_RSQ));
        // owner P = MultiMiMC7([s], 3) = 3 + s + hash(s, 3), kept as a linear combination
        LC s = lc_var(V_KEY), k3; k3[V_ONE] = Fr::from_u32(OWNED_OWNER_KEY);
        LC h = b.perm(s, k3, L.owner_perm);
        LC owner = lc_sum({&k3, &s, &h});
        LC k6, k7; k6[V_ONE] = Fr::from_u32(OWNED_LABELED_PRE_KEY); k7[V_ONE] = Fr::from_u32(OWNED_LABELED_LEAF_KEY);
        LC bl = lc_var(V_BLINDING), tok = lc_var(V_TOKEN), am = lc_var(V_AMOUNT), la = lc_var(V_LABEL);
        b.multi_hash({&owner, &bl}, k6, {L.pre, L.pre + P}, L.pre_out);
        LC vpre = lc_var(L.pre_out);
        b.multi_hash({&vpre, &tok, &am, &la}, k7, {L.leaf, L.leaf + P, L.leaf + 2 * P, L.leaf + 3 * P}, L.leaf_out);
        const uint32_t cur = b.merkle_path(L.leaf_out, L.lvl_base, L.lvl_size, depth);
        // (root - node) * ONE = 0, unconditional: a zero-value note off the tree does not ragequit
        LC vroot = lc_var(V_ROOT), ncur = lc_neg_var(cur);
        b.cs.add(lc_sum({&vroot, &ncur}), lc_var(V_ONE), LC());
        // nullifier = MultiMiMC7([s, leaf, index], 5), the owned labeled transfer's, bound to the public nullifier directly
        LC vleaf = lc_var(L.leaf_out), index, k5; k5[V_ONE] = Fr::from_u32(OWNED_NULLIFIER_KEY);
        Fr pow2 = Fr::one();
        for (uint32_t l = 0; l < depth; l++) {
            lc_add_term(index, L.lvl_base + l * L.lvl_size + 1, pow2);
            pow2 = pow2 + pow2;
        }
        b.multi_hash({&s, &vleaf, &index}, k5, {L.nf_perm, L.nf_perm + P, L.nf_perm + 2 * P}, V_NF);
        return b.cs;
    }
};

// the statement's R1CS at `depth` (ignored by deposit)
inline R1cs statement_r1cs(Statement s, uint32_t depth) {
    switch (s) {
    case ST_WITHDRAW: return WithdrawBuilder::build(depth);
    case ST_DEPOSIT: return DepositBuilder::build();
    case ST_TRANSFER: return TransferBuilder::build(depth);
    case ST_ASSOCIATION: return AssociationBuilder::build(depth);
    case ST_EXCLUSION: return ExclusionBuilder::build(depth);
    case ST_LABELED: return LabeledBuilder::build(depth);
    case ST_LABELED_ASSOCIATION: return LabeledAssociationBuilder::build(depth);
    case ST_OWNED_TRANSFER: return OwnedTransferBuilder::build(depth);
    case ST_OWNED_LABELED_TRANSFER: return OwnedLabeledTransferBuilder::build(depth);
    case ST_RAGEQUIT: return RagequitBuilder::build(depth);
    }
    return R1cs();
}

inline uint32_t groth16_domain_log(uint32_t n_constraints, uint32_t n_pub) {
    uint32_t need = n_constraints + n_pub + 1, k = 0;
    while ((1u << k) < need) k++;
    return k;
}

}  // namespace og
