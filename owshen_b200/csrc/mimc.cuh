// owshen_b200/csrc/mimc.cuh -- declarations of the MiMC7 module and the variable layouts of the
// withdraw, deposit, transfer, association, exclusion, labeled and labeled association withdraw, owned transfer, owned
// labeled transfer and ragequit statements (DESIGN.md section 3; must equal oracle/withdraw_circuit.py: Layout,
// oracle/deposit_circuit.py: Layout, oracle/transfer_circuit.py: Layout, oracle/association_circuit.py: Layout,
// oracle/exclusion_circuit.py: Layout, oracle/labeled_circuit.py: Layout, oracle/labeled_association_circuit.py: Layout,
// oracle/owned_circuit.py: Layout, oracle/owned_labeled_circuit.py: Layout and oracle/ragequit_circuit.py: Layout).
#pragma once
#include <initializer_list>
#include "common.cuh"

namespace og {

constexpr uint32_t WITHDRAW_N_PUB = 3;

struct WithdrawLayout {
    uint32_t depth, perm, cm_base, cm_out, lvl_base, lvl_size, n_vars, n_constraints;
    static WithdrawLayout make(uint32_t depth, uint32_t n_rounds = 91) {
        WithdrawLayout L;
        L.depth = depth;
        L.perm = 4 * n_rounds;
        L.cm_base = 7 + L.perm;
        L.cm_out = L.cm_base + 2 * L.perm;
        L.lvl_base = L.cm_out + 1;
        L.lvl_size = 3 + 2 * L.perm + 1;
        L.n_vars = L.lvl_base + depth * L.lvl_size;
        L.n_constraints = 1 + (L.perm + 1) + (2 * L.perm + 1) + depth * (2 + 2 * L.perm + 1) + 1;
        return L;
    }
};

constexpr uint32_t DEPOSIT_N_PUB = 2;

// 0 ONE | 1 commitment | 2 depositor | 3 nullifier | 4 secret | 5 depositor_sq | 6.. perm1 perm2 out
struct DepositLayout {
    uint32_t perm, cm_base, cm_out, n_vars, n_constraints;
    static DepositLayout make(uint32_t n_rounds = 91) {
        DepositLayout L;
        L.perm = 4 * n_rounds;
        L.cm_base = 6;
        L.cm_out = L.cm_base + 2 * L.perm;
        L.n_vars = L.cm_out + 1;
        L.n_constraints = 1 + (2 * L.perm + 1) + 1;
        return L;
    }
};

constexpr uint32_t TRANSFER_N_PUB = 8;
constexpr uint32_t TRANSFER_AMOUNT_BITS = 64;

// 0 ONE | 1 root | 2 public_amount | 3 token | 4 recipient | 5, 6 nh[2] | 7, 8 out_cm[2] | 9 recipient_sq | 10 nh_diff_inv
// | input blocks 0, 1 | output blocks 0, 1 (oracle/transfer_circuit.py).  A note block starts with nullifier, secret, amount
// and the 64 amount bits; offsets below are relative to the block.
struct TransferLayout {
    uint32_t depth, perm;
    uint32_t in_base, in_size, out_base, out_size;
    uint32_t nh_perm, in_cm, in_cm_out, lvl_base, lvl_size;   // input block
    uint32_t out_cm, out_cm_out;                              // output block
    uint32_t n_vars, n_constraints;
    static TransferLayout make(uint32_t depth, uint32_t n_rounds = 91) {
        TransferLayout L;
        L.depth = depth;
        L.perm = 4 * n_rounds;
        const uint32_t P = L.perm;
        L.lvl_size = 2 * P + 4;
        L.nh_perm = 67; L.in_cm = 67 + P; L.in_cm_out = 67 + 5 * P; L.lvl_base = 68 + 5 * P;
        L.out_cm = 67; L.out_cm_out = 67 + 4 * P;
        L.in_base = 11;
        L.in_size = 68 + 5 * P + depth * L.lvl_size;
        L.out_size = 68 + 4 * P;
        L.out_base = L.in_base + 2 * L.in_size;
        L.n_vars = L.out_base + 2 * L.out_size;
        L.n_constraints = 273 + 18 * P + depth * (4 * P + 6);
        return L;
    }
    OG_HD uint32_t inp(uint32_t i) const { return in_base + i * in_size; }
    OG_HD uint32_t out(uint32_t j) const { return out_base + j * out_size; }
};

// the caller's inputs of a batch of transfers (k_transfer_witness's argument); per proof, input (output) 0 then 1 in the
// in_* (out_*) arrays, in_siblings holds 2 * depth elements (input 0's path, then input 1's) and in_path_bits 2 words
struct TransferInputs {
    const uint8_t *roots, *tokens, *recipients;
    const uint8_t *in_null, *in_sec;
    const uint64_t* in_amounts;
    const uint8_t* in_sib;
    const uint32_t* in_bits;
    const uint8_t *out_null, *out_sec;
    const uint64_t* out_amounts;
};

constexpr uint32_t ASSOCIATION_N_PUB = 4;

// 0 ONE | 1 root | 2 nullifier_hash | 3 recipient | 4 association_root | 5 nullifier | 6 secret | 7 recipient_sq
// | 8.. nullifier-hash permutation | commitment perm1, perm2, out | depth pool levels | depth association levels
// (oracle/association_circuit.py); a level block is the withdraw statement's.
struct AssociationLayout {
    uint32_t depth, perm, cm_base, cm_out, pool_base, assoc_base, lvl_size, n_vars, n_constraints;
    static AssociationLayout make(uint32_t depth, uint32_t n_rounds = 91) {
        AssociationLayout L;
        L.depth = depth;
        L.perm = 4 * n_rounds;
        L.cm_base = 8 + L.perm;
        L.cm_out = L.cm_base + 2 * L.perm;
        L.lvl_size = 2 * L.perm + 4;
        L.pool_base = L.cm_out + 1;
        L.assoc_base = L.pool_base + depth * L.lvl_size;
        L.n_vars = L.assoc_base + depth * L.lvl_size;
        L.n_constraints = 5 + 3 * L.perm + depth * (4 * L.perm + 6);
        return L;
    }
};

// the caller's inputs of a batch of association-set withdrawals (k_association_witness's argument): per proof 32 B each of
// nullifier, secret, recipient, depth siblings per tree and one path-bits word per tree
struct AssociationInputs {
    const uint8_t *nullifiers, *secrets, *recipients, *siblings;
    const uint32_t* path_bits;
    const uint8_t* assoc_siblings;
    const uint32_t* assoc_path_bits;
};

constexpr uint32_t EXCLUSION_N_PUB = 4;
constexpr uint32_t EXCLUSION_RANGE_BITS = 33;

// 0 ONE | 1 root | 2 nullifier_hash | 3 recipient | 4 exclusion_root | 5 nullifier | 6 secret | 7 recipient_sq | 8 low | 9 next
// | 10.. nullifier-hash permutation | commitment perm1, perm2, out | depth pool levels | low, next, gap_lo, gap_hi bits (33 each,
// LSB first) | leaf perm1, perm2, out | depth exclusion levels (oracle/exclusion_circuit.py); a level block is the withdraw
// statement's.
struct ExclusionLayout {
    uint32_t depth, perm, cm_base, cm_out, pool_base, low_bits, next_bits, gap_lo_bits, gap_hi_bits, leaf_base, leaf_out, excl_base,
        lvl_size, n_vars, n_constraints;
    static ExclusionLayout make(uint32_t depth, uint32_t n_rounds = 91) {
        ExclusionLayout L;
        L.depth = depth;
        L.perm = 4 * n_rounds;
        L.cm_base = 10 + L.perm;
        L.cm_out = L.cm_base + 2 * L.perm;
        L.lvl_size = 2 * L.perm + 4;
        L.pool_base = L.cm_out + 1;
        L.low_bits = L.pool_base + depth * L.lvl_size;
        L.next_bits = L.low_bits + EXCLUSION_RANGE_BITS;
        L.gap_lo_bits = L.next_bits + EXCLUSION_RANGE_BITS;
        L.gap_hi_bits = L.gap_lo_bits + EXCLUSION_RANGE_BITS;
        L.leaf_base = L.gap_hi_bits + EXCLUSION_RANGE_BITS;
        L.leaf_out = L.leaf_base + 2 * L.perm;
        L.excl_base = L.leaf_out + 1;
        L.n_vars = L.excl_base + depth * L.lvl_size;
        L.n_constraints = 142 + 5 * L.perm + depth * (4 * L.perm + 6);
        return L;
    }
};

// the caller's inputs of a batch of exclusion withdrawals (k_exclusion_witness's argument): per proof 32 B each of nullifier,
// secret, recipient, depth siblings per tree, one path-bits word per tree, and the keys low, next (u64) of the blocklist leaf
// that brackets the note
struct ExclusionInputs {
    const uint8_t *nullifiers, *secrets, *recipients, *siblings;
    const uint32_t* path_bits;
    const uint64_t *low, *next;
    const uint8_t* excl_siblings;
    const uint32_t* excl_path_bits;
};

constexpr uint32_t LABELED_N_PUB = 7;
constexpr uint32_t LABELED_KEY = 2;            // MultiMiMC7 key of labeled precommitments and leaves (0: commitments, nodes; 1: nullifiers)
constexpr uint32_t LABELED_AMOUNT_BITS = 64, LABELED_LABEL_BITS = 32;

// 0 ONE | 1 root | 2 nullifier_hash | 3 recipient | 4 exclusion_root | 5 token | 6 withdrawn | 7 change_commitment
// | 8 nullifier | 9 secret | 10 recipient_sq | 11 amount | 12 label | 13 change_nullifier | 14 change_secret | 15 low | 16 next
// | 17.. nullifier-hash permutation | precommitment perm1, perm2, out | leaf perm[4], out | depth pool levels
// | amount, withdrawn, change bits (64 each), label bits (32), low, next, gap_lo, gap_hi bits (33 each; all LSB first)
// | change precommitment perm1, perm2, out | change commitment perm[4] | blocklist leaf perm1, perm2, out | depth exclusion
// levels (oracle/labeled_circuit.py); a level block is the withdraw statement's.
struct LabeledLayout {
    uint32_t depth, perm, pre_base, pre_out, leaf_base, leaf_out, pool_base, amount_bits, withdrawn_bits, change_bits, label_bits,
        low_bits, next_bits, gap_lo_bits, gap_hi_bits, cpre_base, cpre_out, ccm_base, xleaf_base, xleaf_out, excl_base, lvl_size,
        n_vars, n_constraints;
    static LabeledLayout make(uint32_t depth, uint32_t n_rounds = 91) {
        LabeledLayout L;
        L.depth = depth;
        L.perm = 4 * n_rounds;
        const uint32_t P = L.perm;
        L.lvl_size = 2 * P + 4;
        L.pre_base = 17 + P;
        L.pre_out = L.pre_base + 2 * P;
        L.leaf_base = L.pre_out + 1;
        L.leaf_out = L.leaf_base + 4 * P;
        L.pool_base = L.leaf_out + 1;
        L.amount_bits = L.pool_base + depth * L.lvl_size;
        L.withdrawn_bits = L.amount_bits + LABELED_AMOUNT_BITS;
        L.change_bits = L.withdrawn_bits + LABELED_AMOUNT_BITS;
        L.label_bits = L.change_bits + LABELED_AMOUNT_BITS;
        L.low_bits = L.label_bits + LABELED_LABEL_BITS;
        L.next_bits = L.low_bits + EXCLUSION_RANGE_BITS;
        L.gap_lo_bits = L.next_bits + EXCLUSION_RANGE_BITS;
        L.gap_hi_bits = L.gap_lo_bits + EXCLUSION_RANGE_BITS;
        L.cpre_base = L.gap_hi_bits + EXCLUSION_RANGE_BITS;
        L.cpre_out = L.cpre_base + 2 * P;
        L.ccm_base = L.cpre_out + 1;
        L.xleaf_base = L.ccm_base + 4 * P;
        L.xleaf_out = L.xleaf_base + 2 * P;
        L.excl_base = L.xleaf_out + 1;
        L.n_vars = L.excl_base + depth * L.lvl_size;
        L.n_constraints = 373 + 15 * P + depth * (4 * P + 6);
        return L;
    }
};

// the caller's inputs of a batch of labeled withdrawals (k_labeled_witness's argument), in C ABI order; per proof: token and
// recipient 32 B each, withdrawn (u64), nullifier and secret 32 B each, amount (u64), label (u32), depth pool siblings and a
// path-bits word, change nullifier and change secret 32 B each, the blocklist leaf's keys low and next (u64), depth
// blocklist-tree siblings and a path-bits word
struct LabeledInputs {
    const uint8_t *tokens, *recipients;
    const uint64_t* withdrawn;
    const uint8_t *nullifiers, *secrets;
    const uint64_t* amounts;
    const uint32_t* labels;
    const uint8_t* siblings;
    const uint32_t* path_bits;
    const uint8_t *change_nullifiers, *change_secrets;
    const uint64_t *low, *next;
    const uint8_t* excl_siblings;
    const uint32_t* excl_path_bits;
};

constexpr uint32_t LABELED_ASSOCIATION_N_PUB = 7;

// 0 ONE | 1 root | 2 nullifier_hash | 3 recipient | 4 association_root | 5 token | 6 withdrawn | 7 change_commitment
// | 8 nullifier | 9 secret | 10 recipient_sq | 11 amount | 12 label | 13 change_nullifier | 14 change_secret | 15 assoc_leaf
// | 16.. nullifier-hash permutation | precommitment perm1, perm2, out | leaf perm[4], out | depth pool levels
// | amount, withdrawn, change bits (64 each), label bits (32; all LSB first) | change precommitment perm1, perm2, out
// | change commitment perm[4] | depth association levels (oracle/labeled_association_circuit.py); a level block is the
// withdraw statement's.  The fields the labeled statement also has mean what they mean in LabeledLayout.
struct LabeledAssociationLayout {
    uint32_t depth, perm, pre_base, pre_out, leaf_base, leaf_out, pool_base, amount_bits, withdrawn_bits, change_bits, label_bits,
        cpre_base, cpre_out, ccm_base, assoc_base, lvl_size, n_vars, n_constraints;
    static LabeledAssociationLayout make(uint32_t depth, uint32_t n_rounds = 91) {
        LabeledAssociationLayout L;
        L.depth = depth;
        L.perm = 4 * n_rounds;
        const uint32_t P = L.perm;
        L.lvl_size = 2 * P + 4;
        L.pre_base = 16 + P;
        L.pre_out = L.pre_base + 2 * P;
        L.leaf_base = L.pre_out + 1;
        L.leaf_out = L.leaf_base + 4 * P;
        L.pool_base = L.leaf_out + 1;
        L.amount_bits = L.pool_base + depth * L.lvl_size;
        L.withdrawn_bits = L.amount_bits + LABELED_AMOUNT_BITS;
        L.change_bits = L.withdrawn_bits + LABELED_AMOUNT_BITS;
        L.label_bits = L.change_bits + LABELED_AMOUNT_BITS;
        L.cpre_base = L.label_bits + LABELED_LABEL_BITS;
        L.cpre_out = L.cpre_base + 2 * P;
        L.ccm_base = L.cpre_out + 1;
        L.assoc_base = L.ccm_base + 4 * P;
        L.n_vars = L.assoc_base + depth * L.lvl_size;
        L.n_constraints = 237 + 13 * P + depth * (4 * P + 6);
        return L;
    }
};

// the caller's inputs of a batch of labeled association withdrawals (k_labeled_association_witness's argument), in C ABI
// order; the first eleven arrays are LabeledInputs', then depth association-tree siblings and a path-bits word per proof
struct LabeledAssociationInputs {
    const uint8_t *tokens, *recipients;
    const uint64_t* withdrawn;
    const uint8_t *nullifiers, *secrets;
    const uint64_t* amounts;
    const uint32_t* labels;
    const uint8_t* siblings;
    const uint32_t* path_bits;
    const uint8_t *change_nullifiers, *change_secrets;
    const uint8_t* assoc_siblings;
    const uint32_t* assoc_path_bits;
};

constexpr uint32_t OWNED_TRANSFER_N_PUB = 8;
// MultiMiMC7 keys of spend-key notes: spend public key P = MultiMiMC7([s], 3), commitment MultiMiMC7([P, blinding, token,
// amount], 4), nullifier MultiMiMC7([s, cm, index], 5)
constexpr uint32_t OWNED_OWNER_KEY = 3, OWNED_COMMITMENT_KEY = 4, OWNED_NULLIFIER_KEY = 5;

// 0 ONE | 1 root | 2 public_amount | 3 token | 4 recipient | 5, 6 nf[2] | 7, 8 out_cm[2] | 9 recipient_sq | 10 nf_diff_inv
// | input blocks 0, 1 | output blocks 0, 1 (oracle/owned_circuit.py).  An input block starts with spend_key, blinding,
// amount and the 64 amount bits, then the owner permutation, the commitment, the depth levels and the nullifier's three
// permutations; an output block is the transfer's with owner in place of nullifier and blinding in place of secret.
// Offsets below are relative to the block.
struct OwnedTransferLayout {
    uint32_t depth, perm;
    uint32_t in_base, in_size, out_base, out_size;
    uint32_t owner_perm, in_cm, in_cm_out, lvl_base, lvl_size, nf_perm;   // input block
    uint32_t out_cm, out_cm_out;                                          // output block
    uint32_t n_vars, n_constraints;
    static OwnedTransferLayout make(uint32_t depth, uint32_t n_rounds = 91) {
        OwnedTransferLayout L;
        L.depth = depth;
        L.perm = 4 * n_rounds;
        const uint32_t P = L.perm;
        L.lvl_size = 2 * P + 4;
        L.owner_perm = 67; L.in_cm = 67 + P; L.in_cm_out = 67 + 5 * P; L.lvl_base = 68 + 5 * P;
        L.nf_perm = L.lvl_base + depth * L.lvl_size;
        L.out_cm = 67; L.out_cm_out = 67 + 4 * P;
        L.in_base = 11;
        L.in_size = 68 + 8 * P + depth * L.lvl_size;
        L.out_size = 68 + 4 * P;
        L.out_base = L.in_base + 2 * L.in_size;
        L.n_vars = L.out_base + 2 * L.out_size;
        L.n_constraints = 273 + 24 * P + depth * (4 * P + 6);
        return L;
    }
    OG_HD uint32_t inp(uint32_t i) const { return in_base + i * in_size; }
    OG_HD uint32_t out(uint32_t j) const { return out_base + j * out_size; }
};

// the caller's inputs of a batch of owned transfers (k_owned_transfer_witness's argument), TransferInputs' shapes: per proof,
// input (output) 0 then 1 in the in_* (out_*) arrays, in_siblings holds 2 * depth elements and in_path_bits 2 words
struct OwnedTransferInputs {
    const uint8_t *roots, *tokens, *recipients;
    const uint8_t *in_keys, *in_blindings;
    const uint64_t* in_amounts;
    const uint8_t* in_sib;
    const uint32_t* in_bits;
    const uint8_t *out_owners, *out_blindings;
    const uint64_t* out_amounts;
};

constexpr uint32_t OWNED_LABELED_TRANSFER_N_PUB = 9;
// MultiMiMC7 keys of owned labeled notes: precommitment MultiMiMC7([P, blinding], 6), leaf MultiMiMC7([pre, token, amount,
// label], 7); the spend public key and the nullifier are the owned notes' (keys 3 and 5)
constexpr uint32_t OWNED_LABELED_PRE_KEY = 6, OWNED_LABELED_LEAF_KEY = 7;

// 0 ONE | 1 root | 2 association_root | 3 token | 4 withdrawn | 5 recipient | 6, 7 nf[2] | 8, 9 out_cm[2] | 10 recipient_sq
// | 11 nf_diff_inv | 12 label | 13 assoc_leaf | 14.. label bits (32) | 46.. withdrawn bits (64) | input blocks 0, 1 | output
// blocks 0, 1 | depth association levels (oracle/owned_labeled_circuit.py).  An input block starts with spend_key, blinding,
// amount and the 64 amount bits, then the owner permutation, the precommitment, the leaf, the depth pool levels and the
// nullifier's three permutations; an output block is owner, blinding, amount, its bits, the precommitment and the leaf.
// Note offsets below are relative to the block; an input's precommitment and leaf sit P later than an output's.
struct OwnedLabeledTransferLayout {
    uint32_t depth, perm;
    uint32_t label_bits, withdrawn_bits;
    uint32_t in_base, in_size, out_base, out_size, assoc_base, lvl_size;
    uint32_t owner_perm, lvl_base, nf_perm;          // input block
    uint32_t pre, pre_out, leaf, leaf_out;           // output block; + perm in an input block
    uint32_t n_vars, n_constraints;
    static OwnedLabeledTransferLayout make(uint32_t depth, uint32_t n_rounds = 91) {
        OwnedLabeledTransferLayout L;
        L.depth = depth;
        L.perm = 4 * n_rounds;
        const uint32_t P = L.perm;
        L.lvl_size = 2 * P + 4;
        L.label_bits = 14;
        L.withdrawn_bits = L.label_bits + LABELED_LABEL_BITS;
        L.pre = 67; L.pre_out = 67 + 2 * P; L.leaf = 68 + 2 * P; L.leaf_out = 68 + 6 * P;
        L.owner_perm = 67; L.lvl_base = 69 + 7 * P;
        L.nf_perm = L.lvl_base + depth * L.lvl_size;
        L.in_base = L.withdrawn_bits + LABELED_AMOUNT_BITS;
        L.in_size = 69 + 10 * P + depth * L.lvl_size;
        L.out_size = 69 + 6 * P;
        L.out_base = L.in_base + 2 * L.in_size;
        L.assoc_base = L.out_base + 2 * L.out_size;
        L.n_vars = L.assoc_base + depth * L.lvl_size;
        L.n_constraints = 377 + 32 * P + depth * (6 * P + 9);
        return L;
    }
    OG_HD uint32_t inp(uint32_t i) const { return in_base + i * in_size; }
    OG_HD uint32_t out(uint32_t j) const { return out_base + j * out_size; }
};

// the caller's inputs of a batch of owned labeled transfers (k_owned_labeled_transfer_witness's argument), in C ABI order;
// per proof: root, token, recipient (32 B each), withdrawn (u64), label (u32), then OwnedTransferInputs' input and output
// arrays, then depth association-tree siblings and a path-bits word
struct OwnedLabeledTransferInputs {
    const uint8_t *roots, *tokens, *recipients;
    const uint64_t* withdrawn;
    const uint32_t* labels;
    const uint8_t *in_keys, *in_blindings;
    const uint64_t* in_amounts;
    const uint8_t* in_sib;
    const uint32_t* in_bits;
    const uint8_t *out_owners, *out_blindings;
    const uint64_t* out_amounts;
    const uint8_t* assoc_sib;
    const uint32_t* assoc_bits;
};

constexpr uint32_t RAGEQUIT_N_PUB = 6;

// 0 ONE | 1 root | 2 token | 3 amount | 4 label | 5 recipient | 6 nullifier | 7 recipient_sq | 8 spend_key | 9 blinding | the
// owner permutation | the precommitment's two permutations and its output | the leaf's four permutations and its output |
// depth pool levels | the nullifier's three permutations (oracle/ragequit_circuit.py).  The owned labeled family's note keys.
struct RagequitLayout {
    uint32_t depth, perm;
    uint32_t owner_perm, pre, pre_out, leaf, leaf_out, lvl_base, lvl_size, nf_perm;
    uint32_t n_vars, n_constraints;
    static RagequitLayout make(uint32_t depth, uint32_t n_rounds = 91) {
        RagequitLayout L;
        L.depth = depth;
        L.perm = 4 * n_rounds;
        const uint32_t P = L.perm;
        L.lvl_size = 2 * P + 4;
        L.owner_perm = 10;
        L.pre = 10 + P; L.pre_out = 10 + 3 * P;
        L.leaf = 11 + 3 * P; L.leaf_out = 11 + 7 * P;
        L.lvl_base = 12 + 7 * P;
        L.nf_perm = L.lvl_base + depth * L.lvl_size;
        L.n_vars = L.nf_perm + 3 * P;
        L.n_constraints = 5 + 10 * P + depth * (2 * P + 3);
        return L;
    }
};

// the caller's inputs of a batch of ragequits (k_ragequit_witness's argument), in C ABI order; per proof: root, token,
// recipient (32 B each), amount (u64), label (u32), spend key, blinding (32 B each), depth siblings and a path-bits word
struct RagequitInputs {
    const uint8_t *roots, *tokens, *recipients;
    const uint64_t* amounts;
    const uint32_t* labels;
    const uint8_t *spend_keys, *blindings, *siblings;
    const uint32_t* path_bits;
};

// ---- the statement table ------------------------------------------------------------------------------------------------
// What the C ABI, the prover and api.py (_STATEMENTS, which mirrors this table) know of a statement.  Besides its row here a
// statement has a layout (above), an R1CS builder (withdraw_circuit.hpp: statement_r1cs), a witness kernel (mimc.cu:
// statement_witness_dev) and its og_* forwarders (capi.cu).
enum Statement : uint32_t { ST_WITHDRAW, ST_DEPOSIT, ST_TRANSFER, ST_ASSOCIATION, ST_EXCLUSION, ST_LABELED, ST_LABELED_ASSOCIATION,
                            ST_OWNED_TRANSFER, ST_OWNED_LABELED_TRANSFER, ST_RAGEQUIT };
constexpr uint32_t STATEMENT_MAX_INPUTS = 15;

struct StatementShape { uint32_t n_vars, n_constraints; };
template <class Layout> StatementShape layout_shape(uint32_t depth) { const Layout L = Layout::make(depth); return {L.n_vars, L.n_constraints}; }
template <> inline StatementShape layout_shape<DepositLayout>(uint32_t) { const DepositLayout L = DepositLayout::make(); return {L.n_vars, L.n_constraints}; }

struct StatementDesc {
    uint32_t n_pub;
    StatementShape (*shape)(uint32_t depth);
    bool takes_depth;                                   // false: one fixed shape, depth 0 throughout
    uint32_t n_inputs;
    // the input arrays in C ABI order: bytes per proof = fixed[k] + per_level[k] * depth
    uint32_t fixed[STATEMENT_MAX_INPUTS], per_level[STATEMENT_MAX_INPUTS];
    uint64_t input_bytes(uint32_t k, uint32_t depth) const { return fixed[k] + (uint64_t)per_level[k] * depth; }
};

constexpr StatementDesc STATEMENTS[] = {
    // withdraw: nullifiers, secrets, recipients, siblings, path_bits
    {WITHDRAW_N_PUB, layout_shape<WithdrawLayout>, true, 5, {32, 32, 32, 0, 4}, {0, 0, 0, 32, 0}},
    // deposit: nullifiers, secrets, depositors
    {DEPOSIT_N_PUB, layout_shape<DepositLayout>, false, 3, {32, 32, 32}, {0, 0, 0}},
    // transfer: roots, tokens, recipients, in_nullifiers, in_secrets, in_amounts, in_siblings, in_path_bits, out_nullifiers,
    // out_secrets, out_amounts
    {TRANSFER_N_PUB, layout_shape<TransferLayout>, true, 11, {32, 32, 32, 64, 64, 16, 0, 8, 64, 64, 16}, {0, 0, 0, 0, 0, 0, 64, 0, 0, 0, 0}},
    // association: nullifiers, secrets, recipients, siblings, path_bits, assoc_siblings, assoc_path_bits
    {ASSOCIATION_N_PUB, layout_shape<AssociationLayout>, true, 7, {32, 32, 32, 0, 4, 0, 4}, {0, 0, 0, 32, 0, 32, 0}},
    // exclusion: nullifiers, secrets, recipients, siblings, path_bits, excl_low, excl_next, excl_siblings, excl_path_bits
    {EXCLUSION_N_PUB, layout_shape<ExclusionLayout>, true, 9, {32, 32, 32, 0, 4, 8, 8, 0, 4}, {0, 0, 0, 32, 0, 0, 0, 32, 0}},
    // labeled: tokens, recipients, withdrawn, nullifiers, secrets, amounts, labels, siblings, path_bits, change_nullifiers,
    // change_secrets, excl_low, excl_next, excl_siblings, excl_path_bits
    {LABELED_N_PUB, layout_shape<LabeledLayout>, true, 15, {32, 32, 8, 32, 32, 8, 4, 0, 4, 32, 32, 8, 8, 0, 4},
     {0, 0, 0, 0, 0, 0, 0, 32, 0, 0, 0, 0, 0, 32, 0}},
    // labeled_association: tokens, recipients, withdrawn, nullifiers, secrets, amounts, labels, siblings, path_bits,
    // change_nullifiers, change_secrets, assoc_siblings, assoc_path_bits
    {LABELED_ASSOCIATION_N_PUB, layout_shape<LabeledAssociationLayout>, true, 13, {32, 32, 8, 32, 32, 8, 4, 0, 4, 32, 32, 0, 4},
     {0, 0, 0, 0, 0, 0, 0, 32, 0, 0, 0, 32, 0}},
    // owned_transfer: roots, tokens, recipients, in_spend_keys, in_blindings, in_amounts, in_siblings, in_path_bits, out_owners,
    // out_blindings, out_amounts
    {OWNED_TRANSFER_N_PUB, layout_shape<OwnedTransferLayout>, true, 11, {32, 32, 32, 64, 64, 16, 0, 8, 64, 64, 16},
     {0, 0, 0, 0, 0, 0, 64, 0, 0, 0, 0}},
    // owned_labeled_transfer: roots, tokens, recipients, withdrawn, labels, in_spend_keys, in_blindings, in_amounts,
    // in_siblings, in_path_bits, out_owners, out_blindings, out_amounts, assoc_siblings, assoc_path_bits
    {OWNED_LABELED_TRANSFER_N_PUB, layout_shape<OwnedLabeledTransferLayout>, true, 15,
     {32, 32, 32, 8, 4, 64, 64, 16, 0, 8, 64, 64, 16, 0, 4}, {0, 0, 0, 0, 0, 0, 0, 0, 64, 0, 0, 0, 0, 32, 0}},
    // ragequit: roots, tokens, recipients, amounts, labels, spend_keys, blindings, siblings, path_bits
    {RAGEQUIT_N_PUB, layout_shape<RagequitLayout>, true, 9, {32, 32, 32, 8, 4, 32, 32, 0, 4}, {0, 0, 0, 0, 0, 0, 0, 32, 0}},
};

// the input arrays of a batch in the statement's C ABI order (host or device pointers)
struct StatementInputs {
    const uint8_t* p[STATEMENT_MAX_INPUTS] = {};
    StatementInputs() = default;
    StatementInputs(std::initializer_list<const void*> xs) {
        uint32_t k = 0;
        for (const void* x : xs) p[k++] = static_cast<const uint8_t*>(x);
    }
    // the same inputs from proof `off` on
    StatementInputs at(Statement s, uint32_t depth, uint32_t off) const {
        StatementInputs r = *this;
        for (uint32_t k = 0; k < STATEMENTS[s].n_inputs; k++) r.p[k] += STATEMENTS[s].input_bytes(k, depth) * off;
        return r;
    }
};

// ---- the note-hash table ------------------------------------------------------------------------------------------------
// The batch hashes of the note families, one thread per item: MultiMiMC7(columns, key).  What the C ABI and api.py
// (_NOTE_HASHES, which mirrors this table) know of a note hash.  Besides its row here a hash has its og_* forwarder (capi.cu);
// mimc.cu's k_note_hash<H> and note_hash_dev serve every row.
enum NoteHash : uint32_t { NH_LABELED_PRECOMMITMENTS, NH_LABELED_LEAVES, NH_OWNED_PUBLIC_KEYS, NH_OWNED_COMMITMENTS, NH_OWNED_NULLIFIERS,
                           NH_OWNED_LABELED_PRECOMMITMENTS, NH_OWNED_LABELED_LEAVES };
// a column's item: a 32-byte canonical field element, or an integer (u64, u32) taken as the field element it is
enum NoteColumn : uint32_t { COL_FR = 32, COL_U64 = 8, COL_U32 = 4 };   // the value is the item's size in bytes
constexpr uint32_t NOTE_HASH_MAX_COLUMNS = 4;

struct NoteHashDesc {
    const char* name;                                   // the kernel's og_profile name
    uint32_t key;                                       // the MultiMiMC7 key
    uint32_t n_cols;
    NoteColumn cols[NOTE_HASH_MAX_COLUMNS];             // the input columns in C ABI order
};

constexpr NoteHashDesc NOTE_HASHES[] = {
    // labeled notes (oracle/labeled_circuit.py): precommitment MultiMiMC7([nullifier, secret], 2), leaf MultiMiMC7([pre, token,
    // amount, label], 2)
    {"k_labeled_precommitments", LABELED_KEY, 2, {COL_FR, COL_FR}},
    {"k_labeled_leaves", LABELED_KEY, 4, {COL_FR, COL_FR, COL_U64, COL_U32}},
    // spend-key notes (oracle/owned_circuit.py): P = MultiMiMC7([s], 3), commitment MultiMiMC7([P, blinding, token, amount], 4),
    // nullifier MultiMiMC7([s, cm, index], 5)
    {"k_owned_public_keys", OWNED_OWNER_KEY, 1, {COL_FR}},
    {"k_owned_commitments", OWNED_COMMITMENT_KEY, 4, {COL_FR, COL_FR, COL_FR, COL_U64}},
    {"k_owned_nullifiers", OWNED_NULLIFIER_KEY, 3, {COL_FR, COL_FR, COL_U32}},
    // owned labeled notes (oracle/owned_labeled_circuit.py): precommitment MultiMiMC7([P, blinding], 6), leaf MultiMiMC7([pre,
    // token, amount, label], 7)
    {"k_owned_labeled_precommitments", OWNED_LABELED_PRE_KEY, 2, {COL_FR, COL_FR}},
    {"k_owned_labeled_leaves", OWNED_LABELED_LEAF_KEY, 4, {COL_FR, COL_FR, COL_U64, COL_U32}},
};

int32_t mimc_hash2_dev(og_ctx* ctx, const uint8_t* d_l, const uint8_t* d_r, uint64_t n, uint8_t* d_out);
int32_t mimc_merkle_paths_dev(og_ctx* ctx, const uint8_t* d_leaves, const uint8_t* d_siblings, const uint32_t* d_bits,
                              uint32_t n_paths, uint32_t depth, uint8_t* d_out);
// the note hash h of n items: cols.p[k] holds column k on the device
int32_t note_hash_dev(og_ctx* ctx, NoteHash h, const StatementInputs& cols, uint64_t n, uint8_t* d_out);
int32_t mimc_to_mont_dev(og_ctx* ctx, const uint8_t* d_in, uint64_t n, Fr* d_out);
int32_t mimc_from_mont_dev(og_ctx* ctx, const Fr* d_in, uint64_t n, uint8_t* d_out);
int32_t mimc_tree_build_dev(og_ctx* ctx, Fr* d_levels, uint64_t n_leaves);
int32_t mimc_tree_append_dev(og_ctx* ctx, uint32_t depth, uint64_t start, uint64_t n, const Fr* h_aux, Fr* d_nodes);
// the statement's witness kernel on device inputs; W rows are w_stride elements apart (the prover keeps two extra scalars
// after every witness)
int32_t statement_witness_dev(og_ctx* ctx, Statement s, uint32_t depth, uint32_t w_stride, const StatementInputs& in, uint32_t batch,
                              Fr* d_W);

// BabyJubJub batch verification (bjj_impl.cuh); out[i] in {0, 1, 2 = public key does not decompress}
int32_t bjj_verify_dev(og_ctx* ctx, const uint8_t* d_pk_x, const uint8_t* d_pk_odd, const uint8_t* d_msgs, const uint8_t* d_sigs,
                       uint32_t n, int hash_kind, uint8_t* d_out);

// batch of PrivateKey::to_pub + sign; status[i] in {1, 2 = "Invalid repr" in the reference}
int32_t bjj_sign_dev(og_ctx* ctx, const uint8_t* d_sk, const uint8_t* d_rnd, const uint8_t* d_msgs, uint32_t n, int hash_kind,
                     uint8_t* d_pk_x, uint8_t* d_pk_odd, uint8_t* d_sigs, uint8_t* d_status);

// encrypted notes (note_impl.cuh; spec oracle/notes.py).  Per note: the recipient's compressed key (pk_x 32 B, pk_odd 1 B),
// nullifier, secret, token (32 B each), amount (u64) and the ephemeral scalar (32 B)
struct NoteEncryptInputs {
    const uint8_t *pk_x, *pk_odd, *nullifiers, *secrets, *tokens;
    const uint64_t* amounts;
    const uint8_t* ephemerals;
};
int32_t note_check_view_keys(og_ctx* ctx, const uint8_t* h_keys, uint32_t n);
int32_t note_public_keys_dev(og_ctx* ctx, const uint8_t* d_keys, uint32_t n, uint8_t* d_pk_x, uint8_t* d_pk_odd);
// The note kinds: NOTE_TRANSFER, commitment key 0.  NOTE_OWNED: spend-key notes (the nullifier and secret fields carry the
// owner P and the blinding), commitment key 4.  NOTE_OWNED_LABELED: owned labeled notes, the owned notes' fields with word 3 =
// amount + 2^64 label (d_labels: one u32 per note, read by this kind only) and the key-7 leaf as commitment (note_core.cuh:
// NOTE_LABELED_KEY).  For the last two a scan's d_spend_keys holds one spend public key P_k per view key (canonical limbs): a
// record is owned by key k only if its m0 is P_k as well.
enum NoteKind : uint32_t { NOTE_TRANSFER, NOTE_OWNED, NOTE_OWNED_LABELED };
OG_HD constexpr uint32_t note_kind_key(NoteKind k) { return k == NOTE_TRANSFER ? 0 : k == NOTE_OWNED ? OWNED_COMMITMENT_KEY : OWNED_LABELED_LEAF_KEY; }
int32_t note_encrypt_dev(og_ctx* ctx, const NoteEncryptInputs& in, uint64_t n, uint8_t* d_records, uint8_t* d_commitments, uint8_t* d_status,
                         NoteKind kind, const uint32_t* d_labels);
int32_t note_scan_dev(og_ctx* ctx, const uint32_t* d_keys, uint32_t n_keys, const uint8_t* d_records, const uint8_t* d_commitments, uint64_t n,
                      uint32_t* d_owner, uint8_t* d_plaintexts, NoteKind kind, const uint32_t* d_spend_keys);

}  // namespace og
