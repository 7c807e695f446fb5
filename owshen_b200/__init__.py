"""owshen_b200 -- H100-native (sm_90a) Groth16 backend for privacy-pool deposit, withdraw, transfer, association-set
withdraw, exclusion withdraw, labeled withdraw, labeled association withdraw, owned transfer, owned labeled transfer and
ragequit proofs over BN254, with encrypted delivery of the notes they create.

Python is the host language here because the reference's (Rust) toolchain is absent from this image;
everything below is a thin ctypes veneer over the C ABI in include/owshen_b200.h, which is the real
drop-in boundary (INTEGRATION.md shows the Rust binding).  There is no CPU fallback: importing works
anywhere, but creating a Context without a CUDA device raises.
"""
from .kvstore import KvStore, MirrorKvStore, RamKvStore
from .api import (Context, ProvingKey, MerkleTree, OwshenB200Error, lib, build_library, prove, verify,
                  setup_withdraw, setup_r1cs, setup_deposit, deposit_r1cs_info, deposit_r1cs_export,
                  setup_transfer, transfer_r1cs_info, transfer_r1cs_export, FR_MODULUS, PROOF_BYTES,
                  setup_association, association_r1cs_info, association_r1cs_export, ptau_prepare_association,
                  ExclusionSet, setup_exclusion, exclusion_r1cs_info, exclusion_r1cs_export, ptau_prepare_exclusion,
                  deposit_labeled, setup_labeled, labeled_r1cs_info, labeled_r1cs_export, ptau_prepare_labeled,
                  ApprovedLabels, setup_labeled_association, labeled_association_r1cs_info, labeled_association_r1cs_export,
                  ptau_prepare_labeled_association,
                  setup_owned_transfer, owned_transfer_r1cs_info, owned_transfer_r1cs_export, ptau_prepare_owned_transfer,
                  deposit_owned_labeled, setup_owned_labeled_transfer, owned_labeled_transfer_r1cs_info,
                  owned_labeled_transfer_r1cs_export, ptau_prepare_owned_labeled_transfer,
                  setup_ragequit, ragequit_r1cs_info, ragequit_r1cs_export, ptau_prepare_ragequit,
                  ptau_new, ptau_contribute, ptau_verify, ptau_prepare, ptau_prepare_withdraw, ptau_prepare_deposit,
                  ptau_prepare_transfer, phase2_contribute, phase2_verify, NOTE_SUBGROUP_ORDER, NOTE_NOT_OWNED, NOTE_MALFORMED)

__all__ = ["Context", "ProvingKey", "MerkleTree", "OwshenB200Error", "lib", "build_library", "prove", "verify",
           "setup_withdraw", "setup_r1cs", "setup_deposit", "deposit_r1cs_info", "deposit_r1cs_export",
           "setup_transfer", "transfer_r1cs_info", "transfer_r1cs_export", "FR_MODULUS", "PROOF_BYTES", "KvStore", "RamKvStore", "MirrorKvStore",
           "ptau_new", "ptau_contribute", "ptau_verify", "ptau_prepare", "ptau_prepare_withdraw", "ptau_prepare_deposit",
           "ptau_prepare_transfer", "phase2_contribute", "phase2_verify",
           "setup_association", "association_r1cs_info", "association_r1cs_export", "ptau_prepare_association",
           "ExclusionSet", "setup_exclusion", "exclusion_r1cs_info", "exclusion_r1cs_export", "ptau_prepare_exclusion",
           "deposit_labeled", "setup_labeled", "labeled_r1cs_info", "labeled_r1cs_export", "ptau_prepare_labeled",
           "ApprovedLabels", "setup_labeled_association", "labeled_association_r1cs_info", "labeled_association_r1cs_export",
           "ptau_prepare_labeled_association",
           "setup_owned_transfer", "owned_transfer_r1cs_info", "owned_transfer_r1cs_export", "ptau_prepare_owned_transfer",
           "deposit_owned_labeled", "setup_owned_labeled_transfer", "owned_labeled_transfer_r1cs_info",
           "owned_labeled_transfer_r1cs_export", "ptau_prepare_owned_labeled_transfer",
           "setup_ragequit", "ragequit_r1cs_info", "ragequit_r1cs_export", "ptau_prepare_ragequit",
           "NOTE_SUBGROUP_ORDER", "NOTE_NOT_OWNED", "NOTE_MALFORMED"]
